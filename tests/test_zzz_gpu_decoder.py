"""GPU parity of row 8f #3 (attention-decoder scoring, CTC prefix scorer, beam loop) -- through the C ABI, against the
fixtures generated from the reference's own TransformerDecoder / CTCPrefixScoreTH / BatchBeamSearch
(tests/golden/decoder_*.npz) and the fp64 oracle.  Bodies and bounds: tests/decoder_gpu_cases.py.

Bounds are pinned at about 4x the errors observed on the GPU."""
import os

import pytest
import torch

import decoder_gpu_cases as cases

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def built():
    assert torch.cuda.is_available(), "run with gpurun"
    import __graft_entry__ as g
    g.build()


@pytest.mark.parametrize("prec", ["fp32", "tf32", "f16"])
@pytest.mark.parametrize("name", ["decoder_tiny", "decoder_full"])
def test_decoder_batch_score_matches_reference_fixture(name, prec):
    cases.batch_score(name, prec)


@pytest.mark.parametrize("prec", ["fp32", "f16"])
def test_decoder_follows_reordered_and_forked_beams(prec):
    cases.forked_beam(prec)


@pytest.mark.parametrize("prec", ["fp32", "f16"])
def test_decoder_long_memory_row_chunks(prec):
    cases.long_memory(prec)


@pytest.mark.parametrize("name", ["decoder_tiny", "decoder_full"])
def test_ctc_prefix_scorer_matches_reference_fixture(name):
    cases.ctc_prefix(name)


@pytest.mark.parametrize("name", ["decoder_tiny", "decoder_full"])
def test_device_beam_search_matches_reference_nbest(name):
    cases.device_beam_search(name)


@pytest.mark.skipif(not os.path.isdir(os.path.join(ROOT, "oracle", "_ref", "espnet")), reason="oracle/_ref did not travel")
def test_reference_batch_beam_search_drives_the_dropins_on_the_gpu():
    cases.reference_loop()


def test_encoder_to_nbest_chain_on_the_dropins():
    cases.encoder_chain()
