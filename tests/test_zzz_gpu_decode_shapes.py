"""GPU checks of the decoding path at the shapes the beam search runs (bodies, size tables and bounds:
tests/decode_shape_cases.py): decoder steps up to 400 positions deep with a beam of 40 that is re-ordered, forked, shrunk
and re-grown, source attention over 1600 frames, the CTC prefix scorer along whole utterances of 1 to 1600 frames, and
the search at bench.py's decode shape.  Yardsticks: the float64 oracle on the same GPU and the reference's own
CTCPrefixScoreTH / BatchBeamSearch from oracle/_ref."""
import pytest
import torch

import decode_shape_cases as cases
from oracle import build_ref

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def built():
    assert torch.cuda.is_available(), "needs a GPU"
    import __graft_entry__ as g
    g.build()


@pytest.fixture(scope="module")
def bk():
    return cases.Backend(dry=False)


@pytest.mark.parametrize("name,prec", [("A1", "fp32"), ("A1", "tf32"), ("A1", "f16"), ("A2", "fp32"), ("A2", "f16"),
                                       ("A3", "fp32"), ("A3", "f16"), ("A4", "fp32"), ("A4", "f16")])
def test_decoder_steps_deep_into_a_prefix_against_float64(bk, name, prec):
    cases.depth(bk, name, prec)


@pytest.mark.parametrize("prec", ["fp32", "f16"])
def test_decoder_step_reads_only_its_chains(bk, prec):
    cases.reads_only_its_chains(bk, "A1", prec)


@pytest.mark.parametrize("prec", ["fp32", "f16"])
def test_decoder_rows_do_not_depend_on_their_order(bk, prec):
    cases.row_order(bk, "A1", prec)


@pytest.mark.parametrize("prec", ["fp32", "f16"])
def test_batched_decoder_rows_at_depth_equal_one_utterance_rows(bk, prec):
    cases.batched_depth(bk, prec)


@pytest.mark.parametrize("T", cases.CTC_SIZES["gpu"]["Ts"])
@pytest.mark.parametrize("kind", ["diffuse", "peaked"])
def test_ctc_prefix_scorer_over_whole_utterances_against_float64(bk, kind, T):
    cases.ctc_whole(bk, kind, T)


def test_batched_ctc_prefix_scorer_over_whole_utterances_equals_one_utterance_scorer(bk):
    cases.ctc_batch_whole(bk)


@pytest.mark.skipif(not build_ref.available(), reason="oracle/_ref did not travel")
@pytest.mark.parametrize("T", [100, 250])
def test_search_matches_reference_search_in_float64(bk, T):
    cases.search(bk, T)
