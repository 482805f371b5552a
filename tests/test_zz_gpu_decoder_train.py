"""GPU parity of the attention decoder's training pass (csrc/decoder_train.cu; TransformerDecoder.forward +
LabelSmoothingLoss, e2e_asr_conformer.py:77-80): against the fixtures generated from the reference's own decoder and
loss in float64 (tests/golden/decoder_train_*.npz), the attention core / label-smoothing / embedding kernels against
float64 restatements on the same GPU, a whole decoder with live attention dropout against the reference with the same
keep-masks, bitwise repeatability, no host synchronisation, the no-grad / eval paths, and the reference E2E.forward with
install() + install_head() + install_decoder() -- which then decodes with the device beam search.

Each test runs in a child process (its own CUDA context).  The bounds are about 4x the errors observed on the H100
(tests/helpers.py record())."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.path.join(ROOT, "oracle", "_ref")
needs_ref = pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "espnet")), reason="oracle/_ref not built")

pytestmark = pytest.mark.gpu

PRELUDE = f"""
import sys, math, importlib.util, numpy as np, torch
sys.path.insert(0, {ROOT!r}); sys.path.insert(0, {HERE!r})
from helpers import record
from auto_avsr_b200 import LabelSmoothingLoss, TransformerDecoder
from auto_avsr_b200 import decoder_train as DT
from oracle import make_golden_decoder_train as M
dev = torch.device("cuda:0")
REF_T = {os.path.join(REF, "espnet", "nets", "pytorch_backend", "transformer")!r}

def ref_module(name):
    spec = importlib.util.spec_from_file_location("_ref_" + name, REF_T + "/" + name + ".py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod

def rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()

def make_batch(ys, odim, mlen, T):
    # add_sos_eos + target_mask + make_non_pad_mask (e2e_asr_conformer.py:67, :77-78)
    eos = odim - 1
    rows = [y[y != -1] for y in ys]
    L = max(len(r) for r in rows) + 1
    ys_in = torch.full((len(rows), L), eos, dtype=torch.long)
    ys_out = torch.full((len(rows), L), -1, dtype=torch.long)
    for b, r in enumerate(rows):
        ys_in[b, 1:len(r) + 1] = r
        ys_out[b, :len(r)] = r
        ys_out[b, len(r)] = eos
    tgt_mask = (ys_in != -1)[:, None, :] & torch.tril(torch.ones(L, L, dtype=torch.bool))[None]
    mem_mask = (torch.arange(T)[None, :] < torch.as_tensor(mlen)[:, None])[:, None, :]
    return ys_in.to(dev), tgt_mask.to(dev), mem_mask.to(dev), ys_out.to(dev)

def golden_case(name, prec, p_att=0.0):
    c = M.CASES[name]
    sd, mem, mlen, ys = M.inputs(name)
    dec = TransformerDecoder(c["odim"], c["d_model"], c["n_heads"], c["linear_units"], c["num_blocks"], dropout_rate=0.0,
                             positional_dropout_rate=0.0, self_attention_dropout_rate=p_att, src_attention_dropout_rate=p_att)
    dec.load_state_dict(sd, strict=True)
    dec = dec.to(dev).train()
    dec.precision = prec
    crit = LabelSmoothingLoss(c["odim"], -1, 0.1, False)
    return dec, crit, mem.to(dev), make_batch(ys, c["odim"], mlen, mem.size(1))

def run(dec, crit, mem, batch):
    ys_in, tgt_mask, mem_mask, ys_out = batch
    x = mem.clone().requires_grad_(True)
    for p in dec.parameters():
        p.grad = None
    pred, _ = dec(ys_in, tgt_mask, x, mem_mask)
    loss = crit(pred, ys_out)
    loss.backward()
    return loss.detach(), pred.detach(), x.grad, {{k: p.grad for k, p in dec.named_parameters()}}

def kbias_scale(key, lookup):
    # softmax is invariant to q . b_k, so d linear_k.bias is 0 up to rounding: measure it against the scale of the same
    # attention's d linear_q.bias instead of its own
    return lookup(key.replace("linear_k.bias", "linear_q.bias")).abs().max().item() if key.endswith("linear_k.bias") else 0.0

def rel_to(a, b, floor):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return ((a - b).abs().max() / max(b.abs().max().item(), floor, 1e-30)).item()

def stored(z, key):
    # -> (reference, function taking the same entries from a whole gradient): the array itself, or its stored subset of
    # rows and columns (steps param_step, or act_step for pred_pad / d memory)
    if key in z.files:
        return torch.as_tensor(z[key]).double(), lambda g: g
    rs, cs = (int(v) for v in z["act_step" if key in ("pred_pad", "d_memory") else "param_step"])
    return torch.as_tensor(z[key + "__rows"]).double(), lambda g: g.reshape(-1, g.shape[-1])[::rs, ::cs]

def stored_err(z, key, got):
    # relative error against a stored array: max-abs for a whole array; for a subset the relative 2-norm error (under
    # TF32 / f16 a ReLU gate of w_1 near 0 can flip against float64: one token's whole contribution to one row, which a
    # max-abs measure over a few stored entries magnifies) and the whole-array checksums [sum, sum |.|, sum of squares].
    # d linear_k.bias is 0 up to rounding (softmax is invariant to q . b_k): it is measured against the scale of the
    # same attention's d linear_q.bias.
    ref, pick = stored(z, key)
    g = pick(got.double().cpu())
    qkey = key.replace("linear_k.bias", "linear_q.bias")
    kb = key.endswith("linear_k.bias")
    if key in z.files:
        return rel_to(g, ref, stored(z, qkey)[0].abs().max().item() if kb else 0.0)
    e = ((g - ref).norm() / max(ref.norm().item(), stored(z, qkey)[0].norm().item() if kb else 0.0, 1e-30)).item()
    cs = z[key + "__checksum"]
    qcs = z[qkey + "__checksum"] if kb else cs
    full = got.double().cpu()
    e_abs = abs(full.abs().sum().item() - cs[1]) / max(cs[1], qcs[1])
    e_sq = abs((full * full).sum().item() - cs[2]) / max(cs[2], qcs[2])
    if max(e, e_abs, e_sq / 2) > 1e-2:
        print("  ", key, "subset", e, "sum|.|", e_abs, "sum^2", e_sq)
    return max(e, e_abs, e_sq / 2)
"""


def run_child(body, timeout=900):
    r = subprocess.run([sys.executable, "-c", PRELUDE + body], capture_output=True, text=True, timeout=timeout, cwd=ROOT)
    assert r.returncode == 0 and "CHILD-OK" in r.stdout, r.stdout[-3000:] + r.stderr[-2500:]


# relative error bounds per precision: loss, logits, d memory, parameter gradients, d feed_forward.w_1.weight.  Under
# TF32 / f16 forward GEMMs a ReLU gate of w_1 close to 0 can flip against float64, which moves one token's whole
# contribution in or out of a row of d w_1: its stored subset of the full case sees 0.07 where every other parameter
# gradient stays within 0.035 (tf32), so w_1 has its own bound.
TOL = {"fp32": (3e-7, 3e-6, 6e-6, 1e-5, 1e-5), "tf32": (3e-4, 5e-3, 3e-2, 0.14, 0.3),
       "f16": (1e-4, 2e-3, 2.5e-2, 0.25, 0.3)}


@pytest.mark.parametrize("name", ["decoder_train_tiny", "decoder_train_full"])
def test_decoder_forward_backward_match_reference_golden(name):
    run_child(f"""
z = np.load(M.GOLDEN + "/" + {name!r} + ".npz")
TOL = {TOL!r}
bad = []
for prec in ("fp32", "tf32", "f16"):
    tl, tp, tm, tg, tw = TOL[prec]
    dec, crit, mem, batch = golden_case({name!r}, prec)
    loss, pred, dmem, grads = run(dec, crit, mem, batch)
    assert tuple(pred.shape) == (mem.size(0), batch[0].size(1), M.CASES[{name!r}]["odim"])
    e_loss = rel(loss, z["loss"])
    e_pred = stored_err(z, "pred_pad", pred)
    e_mem = stored_err(z, "d_memory", dmem)
    e_par = {{k: stored_err(z, "d_" + k, g) for k, g in grads.items()}}
    e_w1 = max(e for k, e in e_par.items() if k.endswith("feed_forward.w_1.weight"))
    worst = max((k for k in e_par if not k.endswith("feed_forward.w_1.weight")), key=e_par.get)
    record("decoder_train_golden", ({name!r}, prec), [e_loss, e_pred, e_mem, e_par[worst], e_w1], [tl, tp, tm, tg, tw])
    print(prec, "worst parameter gradient", worst, e_par[worst], "w_1", e_w1)
    if not (e_loss < tl and e_pred < tp and e_mem < tm and e_par[worst] < tg and e_w1 < tw):
        bad.append((prec, e_loss, e_pred, e_mem, worst, e_par[worst], e_w1))
assert not bad, bad
print("CHILD-OK")
""")


def test_mha_core_matches_fp64_restatement_and_repeats_bitwise():
    run_child("""
def ref_core(q, k, v, H, causal, lengths, keep, scale, dctx):
    B, Lq, D = q.shape
    Lk = k.size(1)
    heads = lambda t: t.double().reshape(B, -1, H, 64).transpose(1, 2).detach().requires_grad_(True)
    qh, kh, vh = heads(q), heads(k), heads(v)
    kl = torch.as_tensor(lengths if lengths is not None else [Lk] * B, device=dev)
    mask = torch.arange(Lk, device=dev)[None, None, None, :] < kl[:, None, None, None]
    if causal:
        mask = mask & (torch.arange(Lk, device=dev)[None, :] <= torch.arange(Lq, device=dev)[:, None])[None, None]
    s = (qh @ kh.transpose(-2, -1) / 8.0).masked_fill(~mask, torch.finfo(torch.float64).min)
    a = torch.softmax(s, -1).masked_fill(~mask, 0.0)
    ad = a if keep is None else a * keep.double() * scale
    out = (ad @ vh).transpose(1, 2).reshape(B, Lq, D)
    (out * dctx.double()).sum().backward()
    back = lambda t: t.transpose(1, 2).reshape(B, -1, D)
    return out.detach(), a.detach(), back(qh.grad), back(kh.grad), back(vh.grad)

cases = [  # (B, H, Lq, Lk, causal, key lengths, p)
    (2, 2, 1, 1, True, None, 0.0),
    (3, 2, 80, 80, True, [80, 37, 0], 0.1),
    (2, 12, 300, 300, True, [300, 211], 0.0),
    (3, 4, 61, 1600, False, [1600, 777, 0], 0.1),
    (2, 3, 1, 450, False, [450, 5], 0.0),
    (2, 2, 300, 1, False, [1, 0], 0.1),
    (5, 12, 80, 400, False, [400, 350, 300, 250, 300], 0.1),
]
g = torch.Generator(device=dev).manual_seed(7)
worst = [0.0] * 5
for B, H, Lq, Lk, causal, lengths, p in cases:
    D = H * 64
    if causal:                                   # self attention: q | k | v slices of one (B, L, 3D) tensor
        src = torch.randn(B, Lq, 3 * D, device=dev, generator=g)
        q, k, v = src[..., :D], src[..., D:2 * D], src[..., 2 * D:]
    else:                                        # source attention: q (B, Lq, D), k | v of one (B, Lk, 2D) tensor
        q = torch.randn(B, Lq, D, device=dev, generator=g)
        kv = torch.randn(B, Lk, 2 * D, device=dev, generator=g) * 2
        k, v = kv[..., :D], kv[..., D:]
    dctx = torch.randn(B, Lq, D, device=dev, generator=g)
    ln = None if lengths is None else torch.tensor(lengths, dtype=torch.int32, device=dev)
    keep = DT.draw_keep_mask(p, (B, H, Lq, Lk), dev) if p > 0 else None
    scale = 1.0 / (1.0 - p)
    outs = []
    for _ in range(2):
        ctx, probs = DT.mha_core_forward(q, k, v, H, causal, ln, keep, scale, want_probs=True)
        ctx_ng, _ = DT.mha_core_forward(q, k, v, H, causal, ln, keep, scale, want_probs=False)
        dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
        DT.mha_core_backward(q, k, v, H, causal, ln, keep, scale, probs, dctx, dq, dk, dv)
        outs.append((ctx, ctx_ng, probs, dq, dk, dv))
    torch.cuda.synchronize()
    for a, b in zip(*outs):
        assert torch.equal(a, b), (B, H, Lq, Lk)
    ctx, ctx_ng, probs, dq, dk, dv = outs[0]
    assert torch.equal(ctx, ctx_ng)
    r = ref_core(q, k, v, H, causal, lengths, keep, scale, dctx)
    gscale = max(t.abs().max().item() for t in r[2:])
    errs = [rel(ctx, r[0]), rel(probs, r[1])] + [rel_to(x, y, gscale) for x, y in zip((dq, dk, dv), r[2:])]
    worst = [max(w, e) for w, e in zip(worst, errs)]
    if lengths is not None and 0 in lengths:
        b0 = lengths.index(0)
        assert (ctx[b0] == 0).all() and (dq[b0] == 0).all() and (dk[b0] == 0).all() and (dv[b0] == 0).all()
bound = [6e-6, 4e-6, 5e-6, 2e-6, 2e-6]
record("mha_core_vs_fp64", "sweep", worst, bound)
assert all(w < b for w, b in zip(worst, bound)), worst
print("CHILD-OK")
""")


@needs_ref
def test_label_smoothing_and_embedding_kernels_match_fp64_and_repeat_bitwise():
    run_child("""
LS = ref_module("label_smoothing_loss")
E = ref_module("embedding")
g = torch.Generator().manual_seed(11)
odim, ld, B, L = 5049, 5056, 5, 81
worst_l, worst_g = 0.0, 0.0
for scale in (1.0, 8.0, 1e4):
    buf = torch.randn(B, L, ld, generator=g) * scale
    buf[..., odim:] = 3e4                                   # padding columns of the padded GEMM output are never read
    if scale == 1e4:
        buf[..., :odim].clamp_(-1e4, 1e4)
    t = torch.randint(0, odim, (B, L), generator=g)
    t[1, 50:] = -1
    t[3, :] = -1                                            # an all-ignored utterance
    x = buf.to(dev)[..., :odim]
    outs = []
    for _ in range(2):
        xg = x.detach().requires_grad_(True)
        loss = DT.label_smoothing_loss(xg, t.to(dev), -1, 0.1)
        (loss * 1.7).backward()
        outs.append((loss.detach(), xg.grad))
    torch.cuda.synchronize()
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    loss, dx = outs[0]
    xr = x.double().cpu().requires_grad_(True)
    ref = LS.LabelSmoothingLoss(odim, -1, 0.1, False)(xr, t)
    (ref * 1.7).backward()
    worst_l = max(worst_l, rel(loss, ref.detach()))
    worst_g = max(worst_g, rel(dx, xr.grad))
    assert (dx[t.to(dev) == -1] == 0).all()
record("label_smoothing_vs_fp64", "ld5056", [worst_l, worst_g], [1e-7, 8e-6])
assert worst_l < 1e-7 and worst_g < 8e-6, (worst_l, worst_g)

# embedding + positional encoding: one token at many positions, fwd / bwd against torch in float64, bitwise repeatable
D = 768
w = torch.randn(odim, D, generator=g)
tok = torch.randint(0, odim, (B, L), generator=g)
tok[:, ::3] = 17
tok[2, :] = 4000
outs = []
for _ in range(2):
    wg = w.to(dev).requires_grad_(True)
    x = DT.EmbedFn.apply(tok.to(dev), wg)
    dy = torch.ones_like(x) * torch.linspace(-1, 1, D, device=dev)
    x.backward(dy)
    outs.append((x.detach(), wg.grad))
torch.cuda.synchronize()
assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
wr = w.double().requires_grad_(True)
ref = E.PositionalEncoding(D, 0.0)(torch.nn.functional.embedding(tok, wr))
ref.backward(torch.ones(B, L, D, dtype=torch.float64) * torch.linspace(-1, 1, D, dtype=torch.float64))
e_x, e_w = rel(outs[0][0], ref.detach()), rel(outs[0][1], wr.grad)
used = torch.zeros(odim, dtype=torch.bool)
used[tok.flatten()] = True
assert (outs[0][1][~used.to(dev)] == 0).all()
bad = torch.tensor([[3, odim]], device=dev)
xb = DT.EmbedFn.apply(bad, w.to(dev))
assert torch.isfinite(xb[0, 0]).all() and torch.isnan(xb[0, 1]).all()
record("embedding_vs_fp64", "odim5049", [e_x, e_w], [3e-7, 6e-6])
assert e_x < 3e-7 and e_w < 6e-6, (e_x, e_w)
print("CHILD-OK")
""")


@needs_ref
def test_decoder_with_attention_dropout_matches_reference_replaying_the_masks():
    run_child(f"""
sys.path.insert(0, {REF!r})
from espnet.nets.pytorch_backend.decoder.transformer_decoder import TransformerDecoder as RefDecoder
from espnet.nets.pytorch_backend.transformer.label_smoothing_loss import LabelSmoothingLoss as RefLS
name = "decoder_train_tiny"
c = M.CASES[name]
dec, crit, mem, batch = golden_case(name, "fp32", p_att=0.1)
drawn = []
orig = DT.draw_keep_mask
def capture(p, shape, device):
    m = orig(p, shape, device)
    drawn.append((p, m))
    return m
DT.draw_keep_mask = capture
loss, pred, dmem, grads = run(dec, crit, mem, batch)
DT.draw_keep_mask = orig
assert len(drawn) == 2 * c["num_blocks"] and all(p == 0.1 for p, _ in drawn)
assert 0.05 < 1.0 - float(torch.cat([m.flatten() for _, m in drawn]).double().mean()) < 0.15

class Replay(torch.nn.Module):                   # the reference's attention dropout, replaying the captured masks in order
    def forward(self, x):
        p, m = drawn.pop(0)
        return x * m.double() / (1.0 - p)
ref = RefDecoder(c["odim"], c["d_model"], c["n_heads"], c["linear_units"], c["num_blocks"], dropout_rate=0.0,
                 positional_dropout_rate=0.0)
ref.load_state_dict(M.inputs(name)[0], strict=True)
ref = ref.double().to(dev).train()
for layer in ref.decoders:
    layer.self_attn.dropout = Replay()
    layer.src_attn.dropout = Replay()
ys_in, tgt_mask, mem_mask, ys_out = batch
xr = mem.double().clone().requires_grad_(True)
pr, _ = ref(ys_in, tgt_mask, xr, mem_mask)
lr = RefLS(c["odim"], -1, 0.1, False)(pr, ys_out)
lr.backward()
assert not drawn
rg = dict(ref.named_parameters())
errs = dict(loss=rel(loss, lr.detach()), pred=rel(pred, pr.detach()), d_memory=rel(dmem, xr.grad))
errs["params"] = max(rel_to(g, rg[k].grad, kbias_scale(k, lambda n: rg[n].grad)) for k, g in grads.items())
record("decoder_dropout_replay_vs_fp64", "tiny", errs, 3e-6)
for k, e in errs.items():
    assert e < 3e-6, (k, e, errs)
print("CHILD-OK")
""")


def test_no_grad_and_eval_equal_train_bitwise_and_no_host_sync():
    run_child("""
for name in ("decoder_train_tiny", "decoder_train_full"):
    dec, crit, mem, batch = golden_case(name, "f16")
    ys_in, tgt_mask, mem_mask, ys_out = batch
    loss_train = run(dec, crit, mem, batch)[0]
    with torch.no_grad():
        pred, _ = dec(ys_in, tgt_mask, mem, mem_mask)
        loss_ng = crit(pred, ys_out)
    dec.eval()
    with torch.no_grad():
        loss_eval = crit(dec(ys_in, tgt_mask, mem, mem_mask)[0], ys_out)
    assert not loss_ng.requires_grad
    assert torch.equal(loss_ng, loss_train) and torch.equal(loss_eval, loss_train), (loss_ng, loss_eval, loss_train)
    dec.train()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    again = run(dec, crit, mem, batch)
    torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert torch.equal(again[0], loss_train)
print("CHILD-OK")
""")


@needs_ref
def test_e2e_with_all_installs_trains_validates_and_decodes_like_reference():
    run_child(f"""
sys.path.insert(0, {REF!r})
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False
from espnet.nets.pytorch_backend.e2e_asr_conformer import E2E
import auto_avsr_b200
from auto_avsr_b200 import shim
odim = 41
torch.manual_seed(0)
ref = E2E(odim, "audio")                   # built before install(): the reference encoder
auto_avsr_b200.install()
ours = E2E(odim, "audio")
ours.load_state_dict(ref.state_dict(), strict=True)
auto_avsr_b200.install_head(ours)
auto_avsr_b200.install_decoder(ours)
assert type(ours.decoder).__module__.startswith("auto_avsr_b200") and type(ours.criterion).__module__.startswith("auto_avsr_b200")
for m in (ref, ours):
    for mod in m.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.p = 0.0
ref = ref.double().to(dev).train()
ours = ours.to(dev).train()
for mod in (ours.encoder, ours.proj_encoder, ours.ctc, ours.decoder):
    mod.precision = "fp32"
g = torch.Generator().manual_seed(5)
lengths = torch.tensor([64, 47]) * 640
x = torch.randn(2, int(lengths.max()), 1, generator=g)
label = torch.randint(1, odim - 1, (2, 9), generator=g)
label[1, 6:] = -1
keys = [k for k, _ in ref.named_parameters() if k.startswith("decoder.")] + [
    "encoder.after_norm.weight", "encoder.after_norm.bias", "frontend.trunk.conv1.weight"]
outs = {{}}
for tag, m, dt in (("ref", ref, torch.float64), ("ours", ours, torch.float32)):
    loss, loss_ctc, loss_att, acc = m(x.to(dev, dt), lengths.to(dev), label.to(dev))
    loss.backward()
    p = dict(m.named_parameters())
    outs[tag] = dict(loss=loss.detach(), loss_ctc=loss_ctc.detach(), loss_att=loss_att.detach(), acc=torch.tensor(acc),
                     **{{k: p[k].grad for k in keys}})
errs = {{k: rel_to(outs["ours"][k], outs["ref"][k], kbias_scale(k, lambda n: outs["ref"][n])) for k in outs["ref"]}}
worst = max(errs, key=errs.get)
record("e2e_all_installs_vs_ref_fp64", "fp32", {{k: errs[k] for k in ("loss", "loss_ctc", "loss_att", "acc", worst)}}, 2e-3)
for k, e in errs.items():
    assert e < 2e-3, (k, e)
# the validation step: eval mode (BatchNorm on running statistics), no autograd
ours.eval()
ref.eval()
with torch.no_grad():
    vloss, _, vatt, vacc = ours(x.to(dev), lengths.to(dev), label.to(dev))
    rloss, _, ratt, racc = ref(x.to(dev, torch.float64), lengths.to(dev), label.to(dev))
e_val = (rel(vloss, rloss), rel(vatt, ratt))
record("e2e_all_installs_validation_vs_ref_fp64", "fp32", list(e_val), 2e-3)
assert max(e_val) < 2e-3 and abs(vacc - racc) < 1e-6, (e_val, vacc, racc)
# and decoding with the same model object
with torch.no_grad():
    feats = ours.frontend(x[:1, :int(lengths[0])].to(dev))
    ids = shim.test_step_decode(ours, feats[0], shim.get_beam_search_decoder(ours, beam_size=3))
assert ids.numel() >= 1, ids
print("decoded", ids.tolist())
print("CHILD-OK")
""", timeout=1500)
