"""The decoding-path checks of tests/decode_shape_cases.py on the host replay (tests/emu: the schedule, slot / ancestor
addressing and every functor of csrc/decoder_body.cuh compiled for the host, fp32) at reduced sizes, against float64:
decoder steps 40 positions deep with a beam that is re-ordered, forked, shrunk and re-grown, and the CTC prefix scorer
driven along whole utterances of 1 / 2 / 3 / 100 frames.  The GPU side is tests/test_zzz_gpu_decode_shapes.py."""
import os

import pytest

import decode_shape_cases as cases
from oracle import build_ref

pytestmark = pytest.mark.skipif(not os.path.exists("/usr/local/cuda/bin/nvcc"), reason="nvcc is needed to build the host replay")


@pytest.fixture(scope="module")
def bk():
    return cases.Backend(dry=True)


def test_decoder_steps_deep_into_a_prefix_against_float64(bk):
    cases.depth(bk, "dry", "fp32")


def test_decoder_single_frame_memory(bk):
    cases.depth(bk, "A4", "fp32")


def test_decoder_step_reads_only_its_chains(bk):
    cases.reads_only_its_chains(bk, "dry", "fp32")


def test_decoder_rows_do_not_depend_on_their_order(bk):
    cases.row_order(bk, "dry", "fp32")


def test_batched_decoder_rows_at_depth_equal_one_utterance_rows(bk):
    cases.batched_depth(bk, "fp32")


@pytest.mark.parametrize("T", cases.CTC_SIZES["dry"]["Ts"])
@pytest.mark.parametrize("kind", ["diffuse", "peaked"])
def test_ctc_prefix_scorer_over_whole_utterances_against_float64(bk, kind, T):
    cases.ctc_whole(bk, kind, T)


def test_batched_ctc_prefix_scorer_over_whole_utterances_equals_one_utterance_scorer(bk):
    cases.ctc_batch_whole(bk)


@pytest.mark.skipif(not build_ref.available(), reason="oracle/_ref is not built")
def test_search_matches_reference_search_in_float64(bk):
    cases.search(bk, 23)
