"""The bf16 precision mode on the GPU: every path that takes a precision, run with precision="bf16" and compared with
float64 and with the f16 mode on the same inputs.

bf16 keeps fp32's 8-bit exponent with a 7-bit mantissa (unit roundoff 2^-8 against f16's 2^-11), so its errors are
expected at about 8x f16's; the bound used below is 16x the f16 error measured in the same test, on the same inputs.
Where a bound is absolute it sits at about 4x the observed value (every comparison is recorded, tests/helpers.py)."""
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch

from helpers import err_stats, load_case, load_head_case, record
from oracle import conformer_oracle as O

pytestmark = pytest.mark.gpu

RATIO = 16.0          # bf16 error <= RATIO x the f16 error on the same inputs (2^3 predicted, 2x slack)
BF16_MAX = 3.3895313892515355e38


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "run with a GPU"
    import __graft_entry__ as g
    g.build()
    return torch.device("cuda:0")


def _edge_values():
    """ties of the bf16 rounding, signed zeros, subnormals, inf / NaN, f16's overflow and bf16's largest finite"""
    ties = [1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8, -(1.0 + 2.0 ** -8), 2.0 ** 100 * (1 + 2.0 ** -8), 1.0 + 2.0 ** -9]
    sub = [1e-40, -1e-40, 2.0 ** -149, -(2.0 ** -149), 2.0 ** -126 * 0.75]
    big = [65504.0 * 4, -65504.0 * 4, 65520.0, BF16_MAX, -BF16_MAX, float(np.nextafter(np.float32(BF16_MAX), np.inf)),
           3.39e38, float(np.finfo(np.float32).max)]
    return torch.tensor(ties + sub + big + [0.0, -0.0, float("inf"), -float("inf"), float("nan")], dtype=torch.float32)


def _same_bits_or_nan(got, want):
    nan = torch.isnan(want.float())
    assert torch.equal(torch.isnan(got.float()), nan)
    assert torch.equal(got[~nan].view(torch.int16), want[~nan].view(torch.int16)), (got[~nan], want[~nan])


# ------------------------------------------------------------------------------------------ 1. operand-exact GEMM
def test_device_conversion_matches_torch_bits(dev):
    """avsr_linear converts x into its bf16 workspace with the library's store: bit for bit torch's rounding (NaN stays
    NaN; its payload is the hardware's canonical one)."""
    from auto_avsr_b200._cabi import lib, check
    from auto_avsr_b200.engine import PRECISIONS
    v = _edge_values()
    k = 64
    x = torch.zeros(1, k)
    x[0, :v.numel()] = v
    w = torch.zeros(8, k)
    nb = int(lib.avsr_linear_workspace_bytes(1, 8, k, PRECISIONS["bf16"]))
    ws = torch.zeros(nb, dtype=torch.uint8, device=dev)
    y = torch.empty(1, 8, device=dev)
    xd, wd = x.to(dev), w.to(dev)
    check(lib.avsr_linear(xd.data_ptr(), wd.data_ptr(), None, None, C.c_float(1.0), 0, y.data_ptr(), 1, 8, k,
                          PRECISIONS["bf16"], ws.data_ptr(), nb, torch.cuda.current_stream(dev).cuda_stream))
    torch.cuda.synchronize()
    got = ws[:2 * k].cpu().view(torch.bfloat16)[:v.numel()]
    _same_bits_or_nan(got, v.to(torch.bfloat16))


@pytest.mark.parametrize("rows,n,k", [(1600, 3072, 768), (1600, 2304, 768), (1600, 1536, 768), (1600, 768, 768),
                                      (1600, 768, 3072), (100, 3072, 768), (100, 768, 3072), (77, 768, 768),
                                      (1, 128, 256)])
def test_linear_operand_exact(dev, rows, n, k):
    """bf16 GEMM vs the float64 product of the bf16-rounded operands: only fp32 accumulation separates them.  The
    same check against f16-rounded operands must miss by >= 10x (the kernel really reads bf16)."""
    from auto_avsr_b200 import ops
    g = torch.Generator().manual_seed(rows + n + k)
    x = torch.randn(rows, k, generator=g)
    w = (torch.rand(n, k, generator=g) * 2 - 1) / math.sqrt(k)
    b = torch.randn(n, generator=g) * 0.1
    y = ops.linear(x.to(dev), w.to(dev), b.to(dev), precision="bf16").cpu().double()
    xb, wb = x.to(torch.bfloat16).double(), w.to(torch.bfloat16).double()
    ref = xb @ wb.T + b.double()
    scale = ref.abs().max().item()
    err = (y - ref).abs().max().item() / scale
    bound = 2e-6 * math.sqrt(k / 768)                  # fp32 accumulation over k products
    record("bf16_linear_exact", (rows, n, k), err, bound)
    assert err < bound, err
    xh, wh = x.half().double(), w.half().double()
    miss = (y - (xh @ wh.T + b.double())).abs().max().item() / scale
    record("bf16_linear_vs_f16_operands", (rows, n, k), miss, 10 * err)
    assert miss >= 10 * err, (miss, err)


def test_linear_operands_entry(dev):
    """avsr_linear_operands with operands already in bf16 storage, fp32 and operand-typed outputs."""
    from auto_avsr_b200._cabi import lib, check
    from auto_avsr_b200.engine import PRECISIONS
    g = torch.Generator().manual_seed(11)
    rows, n, k = 300, 768, 768
    x = torch.randn(rows, k, generator=g).to(torch.bfloat16)
    w = ((torch.rand(n, k, generator=g) * 2 - 1) / math.sqrt(k)).to(torch.bfloat16)
    ref = x.double() @ w.double().T
    st = torch.cuda.current_stream(dev).cuda_stream
    xd, wd = x.to(dev), w.to(dev)
    y = torch.empty(rows, n, device=dev)
    check(lib.avsr_linear_operands(xd.data_ptr(), wd.data_ptr(), None, None, C.c_float(1.0), y.data_ptr(), rows, n, k,
                                   0, 0, PRECISIONS["bf16"], st))
    yo = torch.empty(rows, n, device=dev, dtype=torch.bfloat16)
    check(lib.avsr_linear_operands(xd.data_ptr(), wd.data_ptr(), None, None, C.c_float(1.0), yo.data_ptr(), rows, n, k,
                                   1, 1, PRECISIONS["bf16"], st))
    torch.cuda.synchronize()
    scale = ref.abs().max().item()
    e = (y.cpu().double() - ref).abs().max().item() / scale
    record("bf16_linear_operands", (rows, n, k), e, 2e-6)
    assert e < 2e-6
    # the operand-typed output is the ReLU of the fp32 result rounded once to bf16
    assert torch.equal(yo.cpu(), y.cpu().clamp_min(0).to(torch.bfloat16))


# ------------------------------------------------------------------------------------------ 2. attention
def _attention_err(dev, prec, B, T, H, lengths, g_seed, exact_inputs=False):
    """max error relative to max(1, |ref|) against float64.  exact_inputs: q, k, v, p rounded to bf16 and zero position
    biases, so every input is stored exactly in bf16 and in f16 alike and the error is the kernel's own (P rounded to
    the operand type, fp32 accumulation)"""
    from auto_avsr_b200 import ops
    g = torch.Generator().manual_seed(g_seed)
    D = H * 64
    q, k, v = (torch.randn(B, T, D, generator=g) for _ in range(3))
    p = torch.randn(2 * T - 1, D, generator=g)
    u, vb = torch.randn(H, 64, generator=g) * 0.3, torch.randn(H, 64, generator=g) * 0.3
    if exact_inputs:
        q, k, v, p = (t.to(torch.bfloat16).float() for t in (q, k, v, p))
        u, vb = torch.zeros_like(u), torch.zeros_like(vb)
    ln = None if lengths is None else torch.tensor(lengths, dtype=torch.int32, device=dev)
    ctx = ops.relpos_attention(q.to(dev), k.to(dev), v.to(dev), p.to(dev), u.to(dev), vb.to(dev), ln, H,
                               precision=prec).cpu()

    def heads(t):
        return t.double().view(B, T, H, 64).transpose(1, 2)
    scores = O.rel_attention_scores(heads(q), heads(k), p.double().view(2 * T - 1, H, 64).transpose(0, 1), u.double(),
                                    vb.double())
    if lengths is not None:
        pad = torch.arange(T)[None, :] >= torch.tensor(lengths)[:, None]
        scores = scores.masked_fill(pad[:, None, None, :], float("-inf"))
    attn = torch.softmax(scores, dim=-1)
    attn = torch.where(torch.isnan(attn), torch.zeros_like(attn), attn)
    ref = (attn @ heads(v)).transpose(1, 2).reshape(B, T, D)
    assert torch.isfinite(ctx).all()
    if lengths is not None:
        for b, L in enumerate(lengths):
            if L == 0:
                assert (ctx[b] == 0).all(), "a zero-length utterance has a zero context"
    return err_stats(ctx, ref)[0] / max(1.0, ref.abs().max().item())


@pytest.mark.parametrize("B,T,H,lengths", [(1, 1, 2, None), (2, 63, 4, [63, 40]), (1, 64, 12, None),
                                           (3, 65, 2, [65, 1, 33]), (2, 400, 12, [400, 251]), (1, 1600, 12, None),
                                           (3, 37, 2, [37, 0, 18])])
def test_relpos_attention_within_ratio_of_f16(dev, B, T, H, lengths):
    e16 = _attention_err(dev, "f16", B, T, H, lengths, 5 + T)
    eb = _attention_err(dev, "bf16", B, T, H, lengths, 5 + T)
    bound = RATIO * max(e16, 1e-6)
    record("bf16_attention", (B, T, H, lengths), [eb, e16], bound)
    assert eb < bound, (eb, e16)


@pytest.mark.parametrize("B,T,H,lengths", [(1, 1, 2, None), (2, 65, 4, [65, 33]), (2, 400, 12, [400, 251]),
                                           (1, 1600, 12, None), (3, 37, 2, [37, 0, 18])])
def test_relpos_attention_on_bf16_inputs(dev, B, T, H, lengths):
    """float64 on the bf16-rounded inputs: what is left is the kernel's own error, bf16 <= RATIO x f16"""
    e16 = _attention_err(dev, "f16", B, T, H, lengths, 7 + T, exact_inputs=True)
    eb = _attention_err(dev, "bf16", B, T, H, lengths, 7 + T, exact_inputs=True)
    record("bf16_attention_exact_inputs", (B, T, H, lengths), [eb, e16], RATIO * max(e16, 1e-6))
    assert eb < RATIO * max(e16, 1e-6), (eb, e16)


# ------------------------------------------------------------------------------------------ 3. encoder
def _encoder(case, dev, prec):
    from auto_avsr_b200 import ConformerEncoder
    cfg = case["cfg"]
    enc = ConformerEncoder(attention_dim=cfg["d_model"], attention_heads=cfg["n_heads"],
                           linear_units=cfg["linear_units"], num_blocks=cfg["num_blocks"],
                           cnn_module_kernel=cfg["cnn_kernel"])
    enc.load_state_dict(case["sd"], strict=True)
    enc = enc.to(dev).eval()
    enc.precision = prec
    enc.graph_after = 1
    return enc


def _mask(case, dev):
    return O.non_pad_mask(case["lengths"]).unsqueeze(1).to(dev) if case["masked"] else None


@pytest.mark.parametrize("name", ["full12_ragged", "full12_s1", "full2_ragged", "tiny_ragged"])
def test_encoder_golden_within_ratio_of_f16(dev, name):
    c = load_case(name)
    ref = torch.from_numpy(c["z"]["out_f64"]).double()
    enc = _encoder(c, dev, "f16")
    with torch.no_grad():
        f16_only = enc(c["xs"].to(dev), _mask(c, dev))[0].cpu()
    e16 = err_stats(f16_only, ref)
    outs = {}
    enc.precision = "bf16"
    for graph in (False, True):
        enc.use_graph = graph
        with torch.no_grad():
            outs[graph] = enc(c["xs"].to(dev), _mask(c, dev))[0].cpu()
        eb = err_stats(outs[graph], ref)
        record("bf16_encoder_golden", (name, graph), [eb[0], eb[1], e16[0], e16[1]], RATIO)
        assert torch.isfinite(outs[graph]).all()
        assert eb[0] < RATIO * e16[0] and eb[1] < RATIO * e16[1], (eb, e16)
    assert torch.equal(outs[False], outs[True]), "CUDA-graph replay must be bit-identical to direct launches"
    # the prepared-weight and plan caches key on the precision: f16 after bf16 on the same module = f16 alone
    enc.precision = "f16"
    for graph in (False, True):
        enc.use_graph = graph
        with torch.no_grad():
            again = enc(c["xs"].to(dev), _mask(c, dev))[0].cpu()
        assert torch.equal(again, f16_only), ("f16 after bf16 differs", graph)


def test_per_module_path_agrees_with_fused(dev):
    c = load_case("tiny_ragged")
    enc = _encoder(c, dev, "bf16")
    for m in enc.modules():
        if hasattr(m, "precision"):
            m.precision = "bf16"
    xs, mask = c["xs"].to(dev), _mask(c, dev)
    with torch.no_grad():
        fused = enc(xs, mask)[0].cpu()
        x, pos = enc.embed(xs)
        (x, _), _ = enc.encoders((x, pos), mask)
        y = enc.after_norm(x).cpu()
    ref = torch.from_numpy(c["z"]["out_f64"])
    mx, rms = err_stats(y, ref)
    fmx, frms = err_stats(fused, ref)
    record("bf16_per_module", ("tiny_ragged",), [mx, rms, fmx, frms], [6e-2, 1e-2])
    assert mx < 6e-2 and rms < 1e-2, (mx, rms)
    assert err_stats(y, fused)[0] < 6e-2


@pytest.mark.parametrize("shape", ["S1", "S2", "S2r", "S3", "S4"])
def test_survey_shapes_within_ratio_of_f16(dev, shape):
    from auto_avsr_b200.synthetic import SHAPES, encoder_input, encoder_state_dict
    lengths = list(SHAPES[shape])
    sd = encoder_state_dict(0)
    xs = encoder_input(lengths, 768, 1234)
    case = dict(cfg=dict(d_model=768, n_heads=12, linear_units=3072, num_blocks=12, cnn_kernel=31), sd=sd)
    masked = shape != "S1"
    mask = O.non_pad_mask(lengths).unsqueeze(1).to(dev) if masked else None
    torch.set_num_threads(max(1, torch.get_num_threads()))
    ref = O.encoder_forward(sd, xs.float(), lengths if masked else None, 12)
    errs = {}
    for prec in ("f16", "bf16"):
        enc = _encoder(case, dev, prec)
        with torch.no_grad():
            out = enc(xs.to(dev), mask)[0].cpu()
        assert torch.isfinite(out).all()
        errs[prec] = err_stats(out, ref)
    record("bf16_survey_shapes", (shape,), [*errs["bf16"], *errs["f16"]], RATIO)
    assert errs["bf16"][0] < RATIO * errs["f16"][0] and errs["bf16"][1] < RATIO * errs["f16"][1], errs
    if shape == "S2":
        perm = [3, 1, 0, 2]
        with torch.no_grad():
            outp = enc(xs[perm].to(dev), mask)[0].cpu()
        d = err_stats(outp, out[perm])[0]
        record("bf16_s2_perm", (shape,), d, 2e-2)
        assert d < 2e-2, d


# ------------------------------------------------------------------------------------------ 4. range
def _range_case(scale, w1_only=False):
    from auto_avsr_b200.synthetic import encoder_input, encoder_state_dict
    lengths = [48, 31]
    sd = encoder_state_dict(3, num_blocks=2)
    suffixes = (".w_1.weight",) if w1_only else (".norm_ff.weight", ".norm_ff_macaron.weight", ".w_1.weight",
                                                  ".w_1.bias", ".linear_v.weight")
    for k in list(sd):
        if k.endswith(suffixes):
            sd[k] = sd[k] * scale
    xs = encoder_input(lengths, 768, 7) * (1.0 if w1_only else scale)
    return lengths, sd, xs


def _rel_errs(dev, lengths, sd, xs):
    """(bf16, tf32) errors relative to the output's max-abs; the bf16 forward runs checked and must raise nothing"""
    from auto_avsr_b200 import ConformerEncoder
    ref = O.encoder_forward(sd, xs.double(), lengths, 12)
    enc = ConformerEncoder(num_blocks=2)
    enc.load_state_dict(sd, strict=True)
    enc = enc.to(dev).eval()
    mask = O.non_pad_mask(lengths).unsqueeze(1).to(dev)
    rscale = ref.abs().max().item()
    errs = []
    for prec in ("bf16", "tf32"):
        enc.precision = prec
        enc.check_saturation = prec == "bf16"          # bf16 cannot saturate: the checked forward raises nothing
        with torch.no_grad():
            out = enc(xs.to(dev), mask)[0].cpu()
        assert torch.isfinite(out).all()
        errs.append(err_stats(out, ref)[0] / rscale)
    return errs


def test_range_does_not_cost_relative_accuracy(dev):
    """The scaled weight sets make the problem itself worse conditioned (the relative error of tf32, which has fp32's
    range, grows with the scale too), so range is judged against tf32 on the same set: bf16's error over tf32's error
    stays within 2x of that ratio at scale 1."""
    b1, t1 = _rel_errs(dev, *_range_case(1.0))
    for case in (8.0, 64.0, 1024.0, "w_1 x 2^20"):
        b, t = _rel_errs(dev, *(_range_case(2.0 ** 20, w1_only=True) if isinstance(case, str) else _range_case(case)))
        record("bf16_range", (case,), [b, t, b1, t1], 2.0 * b1 / t1)
        assert b / t < 2.0 * b1 / t1, (case, b, t, b1, t1)


# ------------------------------------------------------------------------------------------ 5. head
def test_head_golden_within_ratio_of_f16(dev):
    from auto_avsr_b200 import CTC, ConformerEncoder, ProjEncoder
    c = load_head_case("head_full")
    cfg, z = c["cfg"], c["z"]
    enc = ConformerEncoder(attention_dim=cfg["d_model"], attention_heads=cfg["n_heads"], linear_units=cfg["linear_units"],
                           num_blocks=cfg["num_blocks"], cnn_module_kernel=cfg["cnn_kernel"])
    enc.load_state_dict(c["enc_sd"], strict=True)
    proj = ProjEncoder(cfg["idim"], cfg["d_model"])
    proj.load_state_dict({"weight": c["head_sd"]["proj_encoder.weight"], "bias": c["head_sd"]["proj_encoder.bias"]})
    ctc = CTC(cfg["odim"], cfg["d_model"], 0.1)
    ctc.load_state_dict({"ctc_lo.weight": c["head_sd"]["ctc.ctc_lo.weight"], "ctc_lo.bias": c["head_sd"]["ctc.ctc_lo.bias"]})
    proj, enc, ctc = (m.to(dev).eval() for m in (proj, enc, ctc))
    mask = O.non_pad_mask(c["lengths"]).unsqueeze(1).to(dev)
    errs = {}
    for prec in ("f16", "bf16"):
        for m in (proj, enc, ctc):
            m.precision = prec
        with torch.no_grad():
            hs, _ = enc(proj(c["feats"].to(dev)), mask)
            logp = ctc.log_softmax(hs)
        errs[prec] = err_stats(logp.cpu(), torch.from_numpy(z["logp_f64"]))
    record("bf16_head_logp", ("head_full",), [*errs["bf16"], *errs["f16"]], RATIO)
    assert errs["bf16"][0] < RATIO * errs["f16"][0] and errs["bf16"][1] < RATIO * errs["f16"][1], errs


def test_ctc_loss_with_bf16_ctc_lo(dev):
    """CTC loss forward / backward through ctc_lo in bf16 vs fp32 mode: finite, and close in relative terms."""
    from auto_avsr_b200 import CTC
    g = torch.Generator().manual_seed(9)
    B, T, D, odim = 3, 60, 768, 41
    hs = torch.randn(B, T, D, generator=g)
    hlens = torch.tensor([60, 44, 31])
    ys = torch.randint(1, odim, (B, 12), generator=g)
    ys[1, 9:] = -1
    ys[2, 5:] = -1
    ctc = CTC(odim, D, 0.0)
    ctc = ctc.to(dev).train()
    res = {}
    for prec in ("fp32", "bf16", "f16"):
        ctc.precision = prec
        ctc.zero_grad()
        h = hs.to(dev).requires_grad_(True)
        loss = ctc(h, hlens.to(dev), ys.to(dev))[0]
        loss.backward()
        torch.cuda.synchronize()
        res[prec] = (loss.detach().cpu().double().reshape(-1), h.grad.cpu().double(), ctc.ctc_lo.weight.grad.cpu().double())
    for prec in ("bf16", "f16"):
        el = abs(res[prec][0] - res["fp32"][0]).max().item() / abs(res["fp32"][0]).max().item()
        eg = max((a - b).abs().max().item() / b.abs().max().item() for a, b in zip(res[prec][1:], res["fp32"][1:]))
        res[prec + "_err"] = (el, eg)
    record("bf16_ctc_loss", ("loss", "grads"), [*res["bf16_err"], *res["f16_err"]], [6e-5, RATIO])
    assert all(torch.isfinite(t).all() for t in res["bf16"])
    # the loss is a sum over frames: its relative error is bounded absolutely (about 4x the observed 1.5e-5 .. 4.5e-5)
    assert res["bf16_err"][0] < 1.8e-4 and res["bf16_err"][1] < RATIO * res["f16_err"][1], res


# ------------------------------------------------------------------------------------------ 6. decoding
def test_device_beam_search_bf16_best_hypothesis(dev):
    """DeviceBeamSearch over the decoder_full fixture with decoder and CTC in bf16: the reference's best hypothesis."""
    import decoder_gpu_cases as D
    from auto_avsr_b200.beam_search import DeviceBeamSearch
    from helpers import load_decoder_case
    c = load_decoder_case("decoder_full")
    cfg = c["cfg"]
    dec, ctc = D._decoder(c, "bf16"), D._ctc(c, "bf16")
    assert dec.precision == "bf16"
    nbest = [h.asdict() for h in DeviceBeamSearch(dec, ctc, beam_size=cfg["beam"], vocab_size=cfg["odim"])(c["memory"].to(dev))]
    L = int(c["z"]["nbest_len_f32"][0])
    gap = abs(nbest[0]["score"] - float(c["z"]["nbest_score_f64"][0]))
    record("bf16_beam_search", ("decoder_full", cfg["beam"]), gap, 5e-2)
    assert nbest[0]["yseq"] == c["z"]["nbest_yseq_f32"][0, :L].tolist()
    assert gap < 5e-2, gap


def test_decoder_steps_deep_into_a_prefix_within_ratio_of_f16(dev):
    """Session A1 of decode_shape_cases (6 layers, d 768, T 100, 40 hypotheses, all 101 positions stepped) against
    float64 at its checked steps, in f16 and in bf16 on the same plan: bf16's worst error <= RATIO x f16's."""
    import decode_shape_cases as cases
    from oracle import decoder_oracle as DO
    bk = cases.Backend(dry=False)
    worst = {}
    for prec in ("f16", "bf16"):
        spec, eng, _, sd64, mem, plan = cases._begin(bk, "A1", prec)
        errs = {}
        for step, _, _, prefixes, _, logp in cases._drive(bk, eng, plan):
            if step not in spec["checked"]:
                continue
            want = DO.decoder_logp(sd64, torch.tensor(prefixes, device=bk.dev), mem.double(), spec["cfg"]["H"])
            assert logp.shape == want.shape and bool(torch.isfinite(logp).all()), (prec, step)
            errs[step] = float((logp.double() - want).abs().max())
        assert sorted(errs) == sorted(spec["checked"])
        worst[prec] = max(errs.values())
    record("bf16_decoder_depth_logp", ("A1",), [worst["bf16"], worst["f16"]], RATIO * worst["f16"])
    assert worst["bf16"] < RATIO * worst["f16"], worst


def test_batched_decoder_rows_equal_one_utterance_rows_bf16(dev):
    """4 utterances decoded in one batched session (the grouped source-attention kernel with its bf16 context store)
    give, bit for bit, the rows of one-utterance sessions"""
    import decode_shape_cases as cases
    cases.batched_depth(cases.Backend(dry=False), "bf16")


# ------------------------------------------------------------------------------------------ 7. front-end
@pytest.mark.parametrize("name", ["frontend_video_88", "frontend_video_t1", "frontend_video_45x61", "frontend_audio_ragged"])
def test_frontend_golden_within_ratio_of_f16(dev, name):
    import os
    from auto_avsr_b200.espnet_dropin.resnet import Conv1dResNet, Conv3dResNet
    from auto_avsr_b200.synthetic import frontend_input, frontend_state_dict
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", name + ".npz"))
    modality = str(z["modality"])
    B, T, H, W = (int(v) for v in z["shape"])
    m = Conv3dResNet() if modality == "video" else Conv1dResNet()
    m.load_state_dict(frontend_state_dict(int(z["wseed"]), modality), strict=True)
    m = m.to(dev).eval()
    x = frontend_input(modality, B, T, H, W, int(z["xseed"])).to(dev)
    ref = torch.from_numpy(z["out_f64"]).double()
    errs = {}
    for prec in ("f16", "bf16"):
        m.precision = prec
        with torch.no_grad():
            y = m(x).cpu().double()
        assert torch.isfinite(y).all()
        errs[prec] = (y - ref).abs().max().item() / ref.abs().max().item()
    record("bf16_frontend_golden", (name,), [errs["bf16"], errs["f16"]], RATIO)
    assert errs["bf16"] < RATIO * errs["f16"], errs


# ------------------------------------------------------------------------------------------ 8. training
def test_ffn_training_past_f16_range(dev):
    """An FFN whose hidden activations exceed 65504: the f16 forward stores them clamped and its gradients go wrong;
    bf16 stores them in range and its gradients stay within the bound of the unscaled case."""
    from auto_avsr_b200.train import LinearFn
    g = torch.Generator().manual_seed(21)
    rows, d, f = 256, 768, 3072
    x = torch.randn(rows, d, generator=g)
    w1 = (torch.rand(f, d, generator=g) * 2 - 1) / math.sqrt(d)
    w2 = (torch.rand(d, f, generator=g) * 2 - 1) / math.sqrt(f)
    dy = torch.randn(rows, d, generator=g)

    def run(scale, prec):
        xs = (x * scale).to(dev).requires_grad_(True)
        a = w1.to(dev).requires_grad_(True)
        b = w2.to(dev).requires_grad_(True)
        h = LinearFn.apply(xs, a, None, True, prec)
        y = LinearFn.apply(h, b, None, False, prec)
        y.backward(dy.to(dev))
        return [t.detach().cpu().double() for t in (y, xs.grad, a.grad, b.grad)], h.detach().abs().max().item()

    def ref(scale):
        xs = (x.double() * scale).requires_grad_(True)
        a, b = w1.double().requires_grad_(True), w2.double().requires_grad_(True)
        y = torch.relu(xs @ a.T) @ b.T
        y.backward(dy.double())
        return [t.detach() for t in (y, xs.grad, a.grad, b.grad)]

    def rel(got, want):
        return max((p - q).abs().max().item() / q.abs().max().item() for p, q in zip(got, want))

    base = rel(run(1.0, "bf16")[0], ref(1.0))
    scale = 2.0 ** 16
    r = ref(scale)
    (gb, hmax) = run(scale, "bf16")
    assert hmax > 65504, hmax
    eb = rel(gb, r)
    e16 = rel(run(scale, "f16")[0], r)
    record("bf16_ffn_past_f16_range", (scale, hmax), [eb, e16, base], [2 * base, 0.1])
    assert eb < 2 * base, (eb, base)
    assert e16 > 0.1, e16          # the f16 step trains on clamped hidden activations


def test_encoder_train_mode_two_layers(dev):
    """The 2-layer encoder in train() (dropouts 0) in bf16 against train_enc2.npz's float64 output and input gradient,
    within RATIO of the f16 mode's errors; the backward stays TF32 in both."""
    import os
    from auto_avsr_b200 import ConformerEncoder
    from auto_avsr_b200.synthetic import encoder_state_dict
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "train_enc2.npz"))
    g = torch.Generator().manual_seed(int(z["seed"]))
    x = torch.randn(3, 37, 768, generator=g, dtype=torch.float64).float()
    r = torch.randn(3, 37, 768, generator=g, dtype=torch.float64).float()
    lengths = [int(v) for v in z["lengths"]]
    mask = O.non_pad_mask(lengths).unsqueeze(1).to(dev)
    errs = {}
    for prec in ("f16", "bf16"):
        enc = ConformerEncoder(num_blocks=2, dropout_rate=0.0, positional_dropout_rate=0.0, attention_dropout_rate=0.0)
        enc.load_state_dict(encoder_state_dict(int(z["wseed"]), 768, 12, 3072, 2, 31), strict=True)
        enc = enc.to(dev).train()
        enc.precision = prec
        xg = x.to(dev).requires_grad_(True)
        y, _ = enc(xg, mask)
        (y * r.to(dev)).sum().backward()
        assert all(torch.isfinite(p.grad).all() for p in enc.parameters() if p.grad is not None)
        ey = (y.detach().cpu().double() - torch.from_numpy(z["y"])).abs().max().item() / np.abs(z["y"]).max()
        ed = (xg.grad.cpu().double() - torch.from_numpy(z["dx"])).abs().max().item() / np.abs(z["dx"]).max()
        errs[prec] = (ey, ed)
    record("bf16_train_enc2", ("y", "dx"), [*errs["bf16"], *errs["f16"]], RATIO)
    assert errs["bf16"][0] < RATIO * errs["f16"][0] and errs["bf16"][1] < RATIO * errs["f16"][1], errs


def test_decoder_training_pass_within_ratio_of_f16():
    """The decoder's teacher-forced training pass (forward, label-smoothing loss, backward) against
    decoder_train_full.npz: loss, logits, d memory and the worst parameter gradient, bf16 <= RATIO x f16"""
    import test_zz_gpu_decoder_train as DTR
    DTR.run_child(f"""
z = np.load(M.GOLDEN + "/decoder_train_full.npz")
errs = {{}}
for prec in ("f16", "bf16"):
    dec, crit, mem, batch = golden_case("decoder_train_full", prec)
    loss, pred, dmem, grads = run(dec, crit, mem, batch)
    e_par = {{k: stored_err(z, "d_" + k, g) for k, g in grads.items()}}
    errs[prec] = [rel(loss, z["loss"]), stored_err(z, "pred_pad", pred), stored_err(z, "d_memory", dmem), max(e_par.values())]
record("bf16_decoder_train_golden", "decoder_train_full", errs, [1e-4, {RATIO!r}, {RATIO!r}, {RATIO!r}])
# the loss is a mean over tokens, where f16's relative error happens to sit at 3.3e-7: it is bounded absolutely, at about
# 4x bf16's observed 2.3e-5 (the same treatment as the CTC loss); logits, d memory and parameter gradients by the ratio
bad = [i for i in range(1, 4) if not errs["bf16"][i] < {RATIO!r} * errs["f16"][i]]
bad += [0] if not errs["bf16"][0] < 1e-4 else []
assert not bad, (bad, errs)
print("CHILD-OK")
""")


@pytest.mark.parametrize("modality", ["video", "audio"])
def test_frontend_library_train_within_ratio_of_f16(dev, modality):
    """The front-end's library training path (wgmma conv units with the raw epilogue, batch-statistics BatchNorm) at the
    bucket shape: output, input-free parameter gradients, bf16 against the fp32 mode within RATIO x f16's deviation"""
    from auto_avsr_b200.espnet_dropin.resnet import Conv1dResNet, Conv3dResNet
    from auto_avsr_b200.synthetic import frontend_input, frontend_state_dict
    shape = (2, 29, 88, 88) if modality == "video" else (2, 16000, 1, 1)
    x = frontend_input(modality, *shape, 3).to(dev)
    res = {}
    for prec in ("fp32", "f16", "bf16"):
        m = Conv3dResNet() if modality == "video" else Conv1dResNet()
        m.load_state_dict(frontend_state_dict(2, modality), strict=True)
        m = m.to(dev).train()
        m.library_train, m.precision = True, prec
        y = m(x)
        g = torch.Generator().manual_seed(8)
        dy = torch.randn(y.shape, generator=g).to(dev)
        (y * dy).sum().backward()
        torch.cuda.synchronize()
        res[prec] = [y.detach().double().cpu()] + [p.grad.double().cpu() for p in m.parameters() if p.grad is not None]
        assert all(torch.isfinite(t).all() for t in res[prec])

    def dev_from_fp32(prec):
        return max((a - b).abs().max().item() / max(b.abs().max().item(), 1e-30) for a, b in zip(res[prec], res["fp32"]))
    eb, e16 = dev_from_fp32("bf16"), dev_from_fp32("f16")
    record("bf16_frontend_library_train", (modality,), [eb, e16], RATIO * e16)
    assert eb < RATIO * e16, (eb, e16)


def test_e2e_with_all_installs_trains_in_bf16():
    """E2E (audio) with install(), install_head, install_decoder and install_frontend(library_train=True), every
    library module in bf16: loss and gradients finite, within RATIO x f16's deviation from the library's fp32 mode"""
    import test_zz_gpu_decoder_train as DTR
    if not os.path.isdir(os.path.join(DTR.REF, "espnet")):
        pytest.skip("oracle/_ref not built")
    DTR.run_child(f"""
sys.path.insert(0, {DTR.REF!r})
from espnet.nets.pytorch_backend.e2e_asr_conformer import E2E
import auto_avsr_b200
odim = 41
torch.manual_seed(0)
auto_avsr_b200.install()
ours = E2E(odim, "audio")
auto_avsr_b200.install_head(ours)
auto_avsr_b200.install_decoder(ours)
auto_avsr_b200.install_frontend(ours, library_train=True)
for mod in ours.modules():
    if isinstance(mod, torch.nn.Dropout):
        mod.p = 0.0
ours = ours.to(dev).train()
state = {{k: v.clone() for k, v in ours.state_dict().items()}}
g = torch.Generator().manual_seed(5)
lengths = torch.tensor([64, 47]) * 640
x = torch.randn(2, int(lengths.max()), 1, generator=g)
label = torch.randint(1, odim - 1, (2, 9), generator=g)
label[1, 6:] = -1
res = {{}}
for prec in ("fp32", "f16", "bf16"):
    ours.load_state_dict(state)
    ours.zero_grad()
    for mod in (ours.encoder, ours.proj_encoder, ours.ctc, ours.decoder, ours.frontend):
        mod.precision = prec
    loss, loss_ctc, loss_att, acc = ours(x.to(dev), lengths.to(dev), label.to(dev))
    loss.backward()
    grads = {{n: p.grad.detach().double().cpu() for n, p in ours.named_parameters() if p.grad is not None}}
    assert len(grads) > 100 and all(torch.isfinite(t).all() for t in grads.values()), prec
    res[prec] = dict(loss=loss.detach().double().cpu(), loss_ctc=loss_ctc.detach().double().cpu(),
                     loss_att=loss_att.detach().double().cpu(), **grads)
def worst(prec):
    return max((res[prec][k] - v).abs().max().item() / max(v.abs().max().item(), 1e-6) for k, v in res["fp32"].items())
eb, e16 = worst("bf16"), worst("f16")
record("bf16_e2e_all_installs_vs_fp32_mode", "bf16", [eb, e16], {RATIO!r} * e16)
assert math.isfinite(eb) and eb < {RATIO!r} * e16, (eb, e16)
print("CHILD-OK")
""", timeout=1500)
