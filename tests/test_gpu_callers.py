"""The reference's CALLERS driving the drop-in on the GPU (VERDICT r01: 'no GPU test goes through the reference's
caller'): auto_avsr_b200.shim replays E2E.forward (e2e_asr_conformer.py:63-71) and ModelModule.test_step
(lightning.py:69-72) line by line; plus the on-device collate of row 8f #4."""
import numpy as np
import pytest
import torch

from helpers import err_stats, record
from oracle import conformer_oracle as O
from oracle import head_oracle as HO

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "run with gpurun"
    import __graft_entry__ as g
    g.build()
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def shell(dev):
    from auto_avsr_b200.shim import E2EShell
    from auto_avsr_b200.synthetic import encoder_state_dict, head_state_dict
    m = E2EShell(elayers=2)
    enc_sd, head_sd = encoder_state_dict(3, num_blocks=2), head_state_dict(3)
    m.encoder.load_state_dict(enc_sd, strict=True)
    m.proj_encoder.load_state_dict({"weight": head_sd["proj_encoder.weight"], "bias": head_sd["proj_encoder.bias"]})
    m.ctc.load_state_dict({"ctc_lo.weight": head_sd["ctc.ctc_lo.weight"], "ctc_lo.bias": head_sd["ctc.ctc_lo.bias"]})
    return m.to(dev).eval(), enc_sd, head_sd


def test_lightning_test_step_replay_twenty_distinct_lengths(dev, shell):
    """config 1: B = 1, masks None, a new T per utterance (lightning.py:72) -- runs on direct launches (no plan built)."""
    from auto_avsr_b200.shim import test_step_encoder
    from auto_avsr_b200.synthetic import frontend_features
    m, enc_sd, head_sd = shell
    Ts = [100, 37, 251, 64, 180, 99, 33, 400, 12, 77, 313, 58, 129, 240, 91, 17, 365, 204, 146, 63]
    with torch.no_grad():
        for T in Ts:
            feats = frontend_features([T], 512, 1000 + T)[0]
            enc_feat = test_step_encoder(m, feats.to(dev))
            assert enc_feat.shape == (T, 768)
            ref = O.encoder_forward(enc_sd, HO.proj_encoder(feats.double().unsqueeze(0), head_sd), None, 12)[0]
            mx, _ = err_stats(enc_feat.cpu(), ref)
            record("test_step_replay", (T,), mx, 1e-2)      # proj_encoder + 2 layers in fp16 operands: observed <= 3.1e-3
            assert mx < 1e-2, (T, mx)
    assert m.encoder._engine.stats["plans_built"] == 0


def test_e2e_forward_replay_matches_oracle(dev, shell):
    from auto_avsr_b200.shim import e2e_forward_encoder
    from auto_avsr_b200.synthetic import frontend_features
    m, enc_sd, head_sd = shell
    lengths = [130, 127, 64, 5]
    feats = frontend_features(lengths, 512, 77)
    with torch.no_grad():
        x, mask = e2e_forward_encoder(m, feats.to(dev), lengths)
        logp = m.ctc.log_softmax(x)
    ref_x = O.encoder_forward(enc_sd, HO.proj_encoder(feats.double(), head_sd), lengths, 12)
    mx, rms = err_stats(x.cpu(), ref_x)
    record("e2e_forward_replay", ("enc",), [mx, rms], [1e-2, 1.2e-3])
    assert mx < 1e-2 and rms < 1.2e-3 and mask.shape == (4, 1, 130)
    ref_lp = HO.ctc_log_softmax(ref_x, head_sd)
    mx, rms = err_stats(logp.cpu(), ref_lp)
    record("e2e_forward_replay", ("logp",), [mx, rms], [5e-3, 1.1e-3])
    assert mx < 5e-3 and rms < 1.1e-3


def test_on_device_collate_matches_the_reference_pad(dev):
    """avsr_pack_padded == datamodule/data_module.py:10-30 `pad` (zero padding to the longest), and its inverse."""
    from auto_avsr_b200.bucketing import max_frames_batches, pack_bucket, unpack_bucket
    rng = np.random.default_rng(3)
    lengths_all = [int(v) for v in rng.integers(5, 400, size=60)]
    batches = max_frames_batches(lengths_all, 1600, 50)
    g = torch.Generator().manual_seed(9)
    for batch in batches[:6]:
        lens = [lengths_all[i] for i in batch]
        utts = [torch.randn(n, 768, generator=g) for n in lens]
        flat = torch.cat(utts).to(dev)
        padded, ln = pack_bucket(flat, lens)
        ref = torch.zeros(len(lens), max(lens), 768)
        for b, u in enumerate(utts):
            ref[b, :u.size(0)] = u
        assert torch.equal(padded.cpu(), ref) and ln.cpu().tolist() == lens
        assert torch.equal(unpack_bucket(padded, lens).cpu(), torch.cat(utts))
