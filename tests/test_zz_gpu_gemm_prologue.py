"""The tensor-core GEMM's static-operand prologue (gemm_tc.cu, EpiParams::b_static).

In the encoder forward and its head, a GEMM whose weight no kernel of the PDL chain writes issues the weight boxes
of its first ring stages, and an L2 prefetch of the whole weight, before griddepcontrol.wait.  That changes when bytes
arrive, never which bytes or the order of any sum, so the outputs must be bit-identical with the prologue off
(AVSR_B200_PROLOGUE=0): the 12-layer encoder at every bucket and 16-bit / tf32 precision, direct launches and the
graph plan.  The pre-wait loads are legal only because the weights are written before
the chain starts: weights re-prepared into the same buffer right before a plan forward, with no host synchronize in
between, must give the forward that follows a full synchronize."""
import contextlib
import ctypes as C
import os

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "needs a CUDA GPU"
    import __graft_entry__ as g
    g.build()
    return torch.device("cuda:0")


@contextlib.contextmanager
def prologue(on: bool):
    old = os.environ.get("AVSR_B200_PROLOGUE")
    os.environ["AVSR_B200_PROLOGUE"] = "1" if on else "0"
    try:
        yield
    finally:
        if old is None:
            os.environ.pop("AVSR_B200_PROLOGUE", None)
        else:
            os.environ["AVSR_B200_PROLOGUE"] = old


def make_encoder(dev, prec, seed=11):
    from auto_avsr_b200 import ConformerEncoder
    from auto_avsr_b200.synthetic import encoder_state_dict
    enc = ConformerEncoder()
    enc.load_state_dict(encoder_state_dict(seed), strict=True)
    enc = enc.to(dev).eval()
    enc.precision = prec
    return enc


@pytest.mark.parametrize("prec", ["f16", "bf16", "tf32"])
@pytest.mark.parametrize("shape", ["S1", "S2", "S2r", "S3", "S4"])
def test_encoder_prologue_same_bits(dev, prec, shape):
    from auto_avsr_b200.synthetic import SHAPES as BUCKETS, encoder_input
    from oracle import conformer_oracle as O
    lengths = BUCKETS[shape]
    xs = encoder_input(lengths, 768, 5).to(dev)
    mask = O.non_pad_mask(lengths).unsqueeze(1).to(dev)

    def fwd(enc, graph):
        enc.use_graph = graph
        with torch.no_grad():
            return enc(xs, mask)[0].clone()
    outs = {}
    for on in (False, True):
        with prologue(on):
            enc = make_encoder(dev, prec)     # a fresh module: its graph plans are captured with this setting
            outs[on] = [fwd(enc, False)] + [fwd(enc, True) for _ in range(3)]
    ref = outs[False][0]
    assert torch.isfinite(ref).all()
    for on in (False, True):
        for i, o in enumerate(outs[on]):
            assert torch.equal(o, ref), (shape, prec, on, i)


def test_reprepared_weights_before_plan_forward(dev):
    """avsr_prepare_weights into the buffer a plan reads, then the plan forward at once on the same stream: the
    forward sees the new weights, exactly as after a synchronize."""
    from auto_avsr_b200._cabi import LAYER_FIELDS, LayerParams, check, lib
    from auto_avsr_b200.engine import PRECISIONS, EncoderEngine
    from auto_avsr_b200.synthetic import SHAPES as BUCKETS, encoder_input, encoder_state_dict
    lengths = BUCKETS["S2"]
    xs = encoder_input(lengths, 768, 5).to(dev)
    lens = torch.tensor(lengths, dtype=torch.int32, device=dev)
    eng = EncoderEngine(768, 12, 3072, 12, 31)
    eng.graph_after = 1
    states = [{k: v.to(dev) for k, v in encoder_state_dict(seed).items()} for seed in (11, 12)]
    buf = eng.prepare(states[0], dev, "f16")
    st = torch.cuda.current_stream(dev).cuda_stream

    def prepare_into(state):
        arr = (LayerParams * 12)()
        for l in range(12):
            for field, suffix in LAYER_FIELDS:
                setattr(arr[l], field, state[f"encoders.{l}.{suffix}"].contiguous().data_ptr())
        check(lib.avsr_prepare_weights(C.byref(eng.cfg), arr, state["after_norm.weight"].data_ptr(),
                                       state["after_norm.bias"].data_ptr(), buf.data_ptr(), eng.prepared_bytes,
                                       PRECISIONS["f16"], st))

    with torch.no_grad():
        first = eng.forward(buf, xs, lens, "f16").clone()            # builds the plan with the first weights
        assert eng.stats["graph"] == 1
        prepare_into(states[1])
        chained = eng.forward(buf, xs, lens, "f16").clone()          # no synchronize in between
        torch.cuda.synchronize()
        after_sync = eng.forward(buf, xs, lens, "f16").clone()
        prepare_into(states[0])
        torch.cuda.synchronize()
        back = eng.forward(buf, xs, lens, "f16").clone()
    assert eng.stats["graph"] == 4
    assert not torch.equal(first, after_sync), "the two weight sets must give different features"
    assert torch.equal(chained, after_sync)
    assert torch.equal(back, first)
