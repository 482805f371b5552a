"""The bf16 backward past the encoder: the tensor-core attention core backward of the decoder
(csrc/decoder_attention_bwd_tc.cu, avsr_mha_core_bwd_tc) against a float64 autograd restatement and against what
torch.autocast(bfloat16) makes of it, its exactness (repeat bits, exact zeros, fp16-overflowing gradients), float64
references with one defect each that must miss it, the whole decoder with ``backward_precision="bf16"`` against the
golden fixtures, and the reference E2E with every knob set against its default backward.

Errors are max-abs differences over the reference's max-abs (for the attention core, over the largest of the three
gradients, as test_mha_core_matches_fp64_restatement_and_repeats_bitwise measures them); bounds are about 4x what the
H100 shows.  Each test runs in a child process (its own CUDA context).

Observed on one H100 80GB HBM3 (700 W): attention-core errors 8e-4 .. 7.7e-3 (bound 3e-2), autocast's 2.9e-3 .. 1.3e-2;
negative controls 0.42 / 2.9 / 0.94 (must be >= 6e-2); E2E with every knob 4.9e-2 (bound 0.2)."""
import pytest

from test_zz_gpu_decoder_train import REF, needs_ref, run_child

pytestmark = pytest.mark.gpu

CORE = """
def ref_core(q, k, v, H, causal, lengths, keep, scale, dctx, dtype=torch.float64):
    # attention.py:59-88 on the projected q / k / v (key mask: finfo.min, softmax, masked_fill 0) under autograd
    B, Lq, D = q.shape
    Lk = k.size(1)
    heads = lambda t: t.to(dtype).reshape(B, -1, H, 64).transpose(1, 2).detach().requires_grad_(True)
    qh, kh, vh = heads(q), heads(k), heads(v)
    kl = torch.as_tensor(lengths if lengths is not None else [Lk] * B, device=dev)
    mask = torch.arange(Lk, device=dev)[None, None, None, :] < kl[:, None, None, None]
    if causal:
        mask = mask & (torch.arange(Lk, device=dev)[None, :] <= torch.arange(Lq, device=dev)[:, None])[None, None]
    s = qh @ kh.transpose(-2, -1) / 8.0
    s = s.masked_fill(~mask, torch.finfo(s.dtype).min)
    a = torch.softmax(s, -1).masked_fill(~mask, 0.0)
    ad = a if keep is None else a * keep.to(a.dtype) * scale
    out = (ad @ vh).transpose(1, 2).reshape(B, Lq, D)
    (out.to(dctx.dtype) * dctx).sum().backward()
    back = lambda t: t.transpose(1, 2).reshape(B, -1, D)
    return back(qh.grad), back(kh.grad), back(vh.grad)

def manual_core(q, k, v, H, causal, lengths, keep, scale, dctx, defect=None):
    # the closed form of decoder_train_body.cuh in float64, with one optional defect: "scale" (the keep-mask without
    # its 1 / (1 - p)), "causal" (the causal flag dropped), "delta" (Delta omitted)
    B, Lq, D = q.shape
    Lk = k.size(1)
    heads = lambda t: t.double().reshape(B, -1, H, 64).transpose(1, 2)
    qh, kh, vh, dc = heads(q), heads(k), heads(v), heads(dctx)
    kl = torch.as_tensor(lengths if lengths is not None else [Lk] * B, device=dev)
    mask = torch.arange(Lk, device=dev)[None, None, None, :] < kl[:, None, None, None]
    if causal and defect != "causal":
        mask = mask & (torch.arange(Lk, device=dev)[None, :] <= torch.arange(Lq, device=dev)[:, None])[None, None]
    a = torch.softmax((qh @ kh.transpose(-2, -1) / 8.0).masked_fill(~mask, -float("inf")), -1).nan_to_num(0.0)
    kf = 1.0 if keep is None else keep.double() * (1.0 if defect == "scale" else scale)
    da = (dc @ vh.transpose(-2, -1)) * kf
    delta = 0.0 if defect == "delta" else (a * da).sum(-1, keepdim=True)
    ds = a * (da - delta) / 8.0
    back = lambda t: t.transpose(1, 2).reshape(B, -1, D)
    return back(ds @ kh), back(ds.transpose(-2, -1) @ qh), back((a * kf).transpose(-2, -1) @ dc)

def make_inputs(B, H, Lq, Lk, causal, p, g, dscale=1.0):
    D = H * 64
    if causal:                                   # self attention: q | k | v slices of one (B, L, 3D) tensor
        src = torch.randn(B, Lq, 3 * D, device=dev, generator=g)
        q, k, v = src[..., :D], src[..., D:2 * D], src[..., 2 * D:]
    else:                                        # source attention: q (B, Lq, D), k | v of one (B, Lk, 2D) tensor
        q = torch.randn(B, Lq, D, device=dev, generator=g)
        kv = torch.randn(B, Lk, 2 * D, device=dev, generator=g) * 2
        k, v = kv[..., :D], kv[..., D:]
    dctx = torch.randn(B, Lq, D, device=dev, generator=g) * dscale
    keep = DT.draw_keep_mask(p, (B, H, Lq, Lk), dev) if p > 0 else None
    return q, k, v, dctx, keep, 1.0 / (1.0 - p)

def library_core(q, k, v, H, causal, ln, keep, scale, dctx):
    # forward (stores the probabilities), then the tensor-core backward into fused gradient buffers like MhaCoreFn's
    ctx, probs = DT.mha_core_forward(q, k, v, H, causal, ln, keep, scale, want_probs=True)
    D = H * 64
    if causal:
        dsrc = torch.full((q.size(0), q.size(1), 3 * D), float("nan"), device=dev)
        dq, dk, dv = dsrc[..., :D], dsrc[..., D:2 * D], dsrc[..., 2 * D:]
    else:
        dq = torch.full(q.shape, float("nan"), device=dev)
        dkv = torch.full((k.size(0), k.size(1), 2 * D), float("nan"), device=dev)
        dk, dv = dkv[..., :D], dkv[..., D:]
    DT.mha_core_backward_tc(q, k, v, H, causal, ln, keep, scale, probs, ctx, dctx, dq, dk, dv)
    return dq, dk, dv

def core_err(got, want):
    gscale = max(t.abs().max().item() for t in want)
    return [rel_to(x, y, gscale) for x, y in zip(got, want)]
"""

CASES = """
cases = [  # (B, H, Lq, Lk, causal, key lengths, p)
    (2, 2, 1, 1, True, None, 0.0),
    (3, 2, 80, 80, True, [80, 37, 0], 0.1),
    (2, 12, 300, 300, True, [300, 211], 0.0),
    (3, 4, 61, 1600, False, [1600, 777, 0], 0.1),
    (2, 3, 1, 450, False, [450, 5], 0.0),
    (2, 2, 300, 1, False, [1, 0], 0.1),
    (5, 12, 80, 400, False, [400, 350, 300, 250, 300], 0.1),
]
"""

BF16_TOL = 3e-2


def test_mha_core_bwd_tc_matches_fp64_and_autocast_and_repeats_bitwise():
    """The case list of the fp32 kernels' test: Lq 1-300, Lk 1-1600, H 2-12, causal self attention and source attention
    on strided fused layouts, key length 0, dropout 0.1.  Two calls give the same bits; a zero-length utterance and the
    keys at or past the key length get exact zeros.  Where the gradients are not degenerate (more than one key), the
    error is also within 2x of torch.autocast(bfloat16) on the same restatement."""
    run_child(CORE + CASES + f"""
TOL = {BF16_TOL!r}
g = torch.Generator(device=dev).manual_seed(7)
worst, worst_auto = [0.0] * 3, [0.0] * 3
for B, H, Lq, Lk, causal, lengths, p in cases:
    q, k, v, dctx, keep, scale = make_inputs(B, H, Lq, Lk, causal, p, g)
    ln = None if lengths is None else torch.tensor(lengths, dtype=torch.int32, device=dev)
    a = library_core(q, k, v, H, causal, ln, keep, scale, dctx)
    b = library_core(q, k, v, H, causal, ln, keep, scale, dctx)
    torch.cuda.synchronize()
    for x, y in zip(a, b):
        assert torch.isfinite(x).all() and torch.equal(x, y), (B, H, Lq, Lk)
    dq, dk, dv = a
    want = ref_core(q, k, v, H, causal, lengths, keep, scale, dctx.double())
    errs = core_err(a, want)
    record("mha_core_bwd_tc_vs_fp64", (B, H, Lq, Lk, causal, p), errs, TOL)
    worst = [max(w, e) for w, e in zip(worst, errs)]
    for b_, L in enumerate(lengths or []):
        assert not dk[b_, L:].any() and not dv[b_, L:].any(), (B, H, Lq, Lk, b_)
        if L == 0:
            assert not dq[b_].any(), (B, H, Lq, Lk)
    if Lk > 1 and Lq > 1:
        with torch.autocast("cuda", dtype=torch.bfloat16):
            mixed = ref_core(q, k, v, H, causal, lengths, keep, scale, dctx, dtype=torch.float32)
        e_auto = core_err([t.float() for t in mixed], want)
        record("mha_core_bwd_tc_autocast_error", (B, H, Lq, Lk, causal, p), e_auto, TOL)
        worst_auto = [max(w, e) for w, e in zip(worst_auto, e_auto)]
        assert all(e <= 2 * ea for e, ea in zip(errs, e_auto)), (B, H, Lq, Lk, errs, e_auto)
print("worst", worst, "autocast", worst_auto)
assert all(w < TOL for w in worst), worst
print("CHILD-OK")
""")


def test_mha_core_bwd_tc_range_and_negative_controls():
    """dctx x 2^20: gradients pass fp16's 65504 and stay finite within the bound (bf16 keeps fp32's range).  Float64
    references with one defect each (no keep scale, the causal flag dropped, Delta omitted) must miss the library by at
    least 2x the bound; the defect-free closed form agrees with the autograd restatement first."""
    run_child(CORE + f"""
TOL = {BF16_TOL!r}
g = torch.Generator(device=dev).manual_seed(11)
B, H, Lq, Lk, lengths = 2, 4, 130, 130, [130, 100]
ln = torch.tensor(lengths, dtype=torch.int32, device=dev)
q, k, v, dctx, keep, scale = make_inputs(B, H, Lq, Lk, True, 0.3, g, dscale=2.0 ** 20)
got = library_core(q, k, v, H, True, ln, keep, scale, dctx)
want = ref_core(q, k, v, H, True, lengths, keep, scale, dctx.double())
assert max(t.abs().max().item() for t in got) > 65504
errs = core_err(got, want)
record("mha_core_bwd_tc_range", (B, H, Lq, Lk), errs, TOL)
assert all(torch.isfinite(t).all() for t in got) and max(errs) < TOL, errs
clean = manual_core(q, k, v, H, True, lengths, keep, scale, dctx)
assert max(core_err(clean, want)) < 1e-10
for defect in ("scale", "causal", "delta"):
    e = max(core_err(got, manual_core(q, k, v, H, True, lengths, keep, scale, dctx, defect)))
    record("mha_core_bwd_tc_negative_control", (defect,), e, 2 * TOL)
    assert e >= 2 * TOL, (defect, e)
print("CHILD-OK")
""")


# bounds per forward precision on the golden fixtures, with the bf16 backward: loss, logits, d memory, parameter
# gradients, d feed_forward.w_1.weight (the stored_err measure of test_decoder_forward_backward_match_reference_golden)
# (observed on the H100 at 700 W, worst of the tiny and full fixtures: f16 2.2e-5 / 3.8e-4 / 6.4e-3 / 5.9e-2 / 7.4e-2,
# bf16 8.1e-5 / 3.2e-3 / 1.4e-2 / 8.6e-2 / 8.7e-2)
TOL_BF16_BWD = {"f16": (1e-4, 2e-3, 2.5e-2, 0.25, 0.3), "bf16": (3.5e-4, 1.3e-2, 6e-2, 0.35, 0.35)}


@pytest.mark.parametrize("name", ["decoder_train_tiny", "decoder_train_full"])
def test_decoder_bf16_backward_matches_golden(name):
    """The whole decoder + LabelSmoothingLoss with backward_precision="bf16" at f16 and bf16 forward precision against
    the float64 fixtures of the reference; the loss and logits are the default backward's bits (the forward is
    unchanged)."""
    run_child(f"""
z = np.load(M.GOLDEN + "/" + {name!r} + ".npz")
TOL = {TOL_BF16_BWD!r}
bad = []
for prec in ("f16", "bf16"):
    tl, tp, tm, tg, tw = TOL[prec]
    dec, crit, mem, batch = golden_case({name!r}, prec)
    loss0, pred0, _, _ = run(dec, crit, mem, batch)
    dec.backward_precision = "bf16"
    loss, pred, dmem, grads = run(dec, crit, mem, batch)
    assert torch.equal(loss, loss0) and torch.equal(pred, pred0)
    assert torch.isfinite(dmem).all() and all(torch.isfinite(g).all() for g in grads.values())
    e_loss = rel(loss, z["loss"])
    e_pred = stored_err(z, "pred_pad", pred)
    e_mem = stored_err(z, "d_memory", dmem)
    e_par = {{k: stored_err(z, "d_" + k, g) for k, g in grads.items()}}
    e_w1 = max(e for k, e in e_par.items() if k.endswith("feed_forward.w_1.weight"))
    worst = max((k for k in e_par if not k.endswith("feed_forward.w_1.weight")), key=e_par.get)
    record("decoder_bf16_backward_golden", ({name!r}, prec), [e_loss, e_pred, e_mem, e_par[worst], e_w1], [tl, tp, tm, tg, tw])
    print(prec, "worst parameter gradient", worst, e_par[worst], "w_1", e_w1)
    if not (e_loss < tl and e_pred < tp and e_mem < tm and e_par[worst] < tg and e_w1 < tw):
        bad.append((prec, e_loss, e_pred, e_mem, worst, e_par[worst], e_w1))
assert not bad, bad
print("CHILD-OK")
""")


def test_decoder_knob_cleared_matches_never_set():
    """A decoder whose knob was set to "bf16" and cleared again gives the bits of one that never set it."""
    run_child("""
dec, crit, mem, batch = golden_case("decoder_train_full", "f16")
never = run(dec, crit, mem, batch)
dec.backward_precision = "bf16"
run(dec, crit, mem, batch)
dec.backward_precision = None
again = run(dec, crit, mem, batch)
for a, b in zip(never[:3], again[:3]):
    assert torch.equal(a, b)
for k in never[3]:
    assert torch.equal(never[3][k], again[3][k]), k
print("CHILD-OK")
""")


E2E_TOL = 0.2      # observed 4.9e-2 on the H100 (700 W): encoder.encoders.0.self_attn.pos_bias_v


@needs_ref
def test_e2e_all_knobs_bf16_close_to_default_backward():
    """The reference E2E with install() + install_head() + install_decoder() and backward_precision="bf16" on the
    encoder, proj_encoder, the CTC head and the decoder: every parameter gradient and the gradient of the front-end
    features entering proj_encoder within E2E_TOL of the default backward's, relative to each tensor's max (linear_k's
    bias, which is mathematically 0, against the scale of linear_q's)."""
    run_child(f"""
sys.path.insert(0, {REF!r})
from espnet.nets.pytorch_backend.e2e_asr_conformer import E2E
import auto_avsr_b200
odim = 41
torch.manual_seed(0)
auto_avsr_b200.install()
model = E2E(odim, "audio")
auto_avsr_b200.install_head(model)
auto_avsr_b200.install_decoder(model)
for mod in model.modules():
    if isinstance(mod, torch.nn.Dropout):
        mod.p = 0.0
model = model.to(dev).train()
sd = {{k: v.clone() for k, v in model.state_dict().items()}}
g = torch.Generator().manual_seed(5)
lengths = torch.tensor([64, 47]) * 640
x = torch.randn(2, int(lengths.max()), 1, generator=g).to(dev)
label = torch.randint(1, odim - 1, (2, 9), generator=g)
label[1, 6:] = -1
feats = {{}}
model.proj_encoder.register_forward_pre_hook(lambda m, a: (a[0].retain_grad(), feats.__setitem__("x", a[0])) and None)
grads = {{}}
for backward in (None, "bf16"):
    model.load_state_dict(sd)                  # the same BatchNorm running statistics in both runs
    model.zero_grad(set_to_none=True)
    for mod in (model.encoder, model.proj_encoder, model.ctc, model.decoder):
        mod.backward_precision = backward
    loss = model(x, lengths.to(dev), label.to(dev))[0]
    loss.backward()
    assert torch.isfinite(loss)
    grads[backward] = {{"features": feats["x"].grad, **{{k: p.grad for k, p in model.named_parameters()}}}}
errs = {{}}
for k, g0 in grads[None].items():
    g1 = grads["bf16"][k]
    assert g1 is not None and torch.isfinite(g1).all(), k
    if k.endswith("depthwise_conv.bias"):      # a bias in front of BatchNorm: mathematically 0
        continue
    errs[k] = rel_to(g1, g0, kbias_scale(k, lambda n: grads[None][n]))
worst = max(errs, key=errs.get)
print("worst", worst, errs[worst], "features", errs["features"])
record("e2e_all_knobs_bf16_vs_default", ("worst", worst), errs[worst], {E2E_TOL!r})
assert errs[worst] < {E2E_TOL!r}, (worst, errs[worst])
print("CHILD-OK")
""", timeout=1500)
