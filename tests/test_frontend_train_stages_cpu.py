"""Without a GPU: the case list of tests/test_zz_gpu_frontend_train_stages.py reaches every edge of the training
kernels it is there for, and the float64 unit oracle (oracle/frontend_train_stages.py) is torch's own unit, each of
its defects changes it, and its winner-pinned max-pool is torch's max-pool when the winners agree.

The wgrad split counts come from the library itself: ``avsr_frontend_train_wgrad_workspace_bytes`` is
splits * C_out * Kw * 4 bytes + 256 (Kw = K rounded up to 64), so a change of the split rule shows up here; so do the
BatchNorm statistics tiles (``avsr_bn_train_workspace_bytes``) against the oracle's tile rule."""
import pytest
import torch

from oracle import frontend_train_stages as S


def _splits(g):
    from auto_avsr_b200._cabi import lib
    Kw = -(-g.K // S.WG_T) * S.WG_T
    b = lib.avsr_frontend_train_wgrad_workspace_bytes(*g.args())
    assert b > 256 and (b - 256) % (g.Cout * Kw * 4) == 0, (g.name, b)
    return (b - 256) // (g.Cout * Kw * 4)


def _stats_tiles(g):
    """avsr_bn_train_workspace_bytes is tiles * 3 * C * 8 bytes + 256 (exact for C a multiple of 64)"""
    from auto_avsr_b200._cabi import lib
    return (lib.avsr_bn_train_workspace_bytes(g.rows, g.Cout) - 256) // (3 * g.Cout * 8)


def _all_units(prec=None):
    for case in S.CASES:
        if prec is None or prec in case[7]:
            for g in S.units(case):
                yield case, g


def test_case_list_reaches_every_edge():
    seen = set()
    for case, g in _all_units():
        s = _splits(g)
        ranges = g.split_ranges(s)
        tc = any(p != "fp32" for p in case[7])
        if tc and s > 1:
            seen.add(("tc_multi_split", g.Cout))
        if ranges[-1][0] == ranges[-1][1]:
            seen.add("empty_trailing_split")
        hw = g.Ho * g.Wo
        for lo, hi in ranges[1:]:
            if 0 < lo < g.rows and lo % hw:
                seen.add("split_mid_frame")
                if g.stem == 1 and g.T > 1 and (lo // hw) % g.T:
                    seen.add("stem_split_mid_utterance")
        if g.stem in (1, 2) and g.K % 64:
            seen.add(("k_not_multiple_of_64", g.stem))
        if g.stem == 0 and g.stride == 2 and g.dims == 2:
            seen.add(("dgrad_s2", g.H % 2, g.W % 2))
            if g.KH == 1:
                seen.add("downsample_zero_classes")
        if g.stem == 0 and g.dims == 1 and g.stride == 2:
            seen.add("audio_h1_dgrad")
        tile = S.stats_tile_rows(g.rows, g.Cout)
        assert _stats_tiles(g) == -(-g.rows // tile), (g.name, g.rows, g.Cout)
        if g.rows % tile in (1, tile - 1):
            seen.add(("stats_tail", "1 row" if g.rows % tile == 1 else "1 row short"))
        if g.name.startswith("layer4") and g.rows <= 32 and case[1] == "video":
            seen.add("layer4_bn_le_32")
    want = {("tc_multi_split", c) for c in (64, 128, 256, 512)} | {
        "empty_trailing_split", "split_mid_frame", "stem_split_mid_utterance", ("k_not_multiple_of_64", 1),
        ("k_not_multiple_of_64", 2), ("dgrad_s2", 0, 0), ("dgrad_s2", 1, 1), "downsample_zero_classes",
        "audio_h1_dgrad", ("stats_tail", "1 row"), ("stats_tail", "1 row short"), "layer4_bn_le_32"}
    assert want <= seen, sorted(map(str, want - seen))


def test_bucket_split_counts():
    """The split counts the bucket cases are in the list for (the video stem 132 x 23,488 pixels, the layer-3
    downsample's last split empty, 17 layer-4 downsample splits; 42 frames: layer 1's last split empty, 4 of the
    stem's)."""
    by = {(c[0], c[1], g.name): g for c, g in _all_units()}
    stem = by[("bucket", "video", "stem")]
    assert _splits(stem) == 132 and stem.split_rows(132) == 23488
    ds3 = by[("bucket", "video", "layer3.0.downsample")]
    assert _splits(ds3) == 66 and ds3.split_ranges(66)[-1][0] == ds3.rows
    assert _splits(by[("bucket", "video", "layer4.0.downsample")]) == 17
    l1 = by[("t7_42", "video", "layer1.0.conv1")]
    assert _splits(l1) == 59 and l1.split_ranges(59)[-1][0] == l1.rows
    st = by[("t7_42", "video", "stem")]
    assert sum(lo == hi for lo, hi in st.split_ranges(_splits(st))) == 4


def _unit_inputs(g, resid, seed=0):
    gen = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=gen, dtype=torch.float64)
    if g.stem == 1:
        x, w = r(g.N, g.H, g.W), r(64, 1, 5, 7, 7) / 15
    elif g.stem == 2:
        x, w = r(g.N, g.W), r(64, 1, 80) / 9
    else:
        x = r(g.N, g.H, g.W, g.Cin) + 0.5
        w = (r(g.Cout, g.Cin, g.KH, g.KW) if g.dims == 2 else r(g.Cout, g.Cin, g.KW)) / (g.K ** 0.5)
    out = (g.N, g.Ho, g.Wo, g.Cout)
    return (x, r(*out) if resid else None, w, 1 + 0.2 * r(g.Cout), 0.2 * r(g.Cout), 0.1 * r(g.Cout),
            1 + r(g.Cout).abs(), 0.1, 1e-5, g), r(*out)


TINY = [S.Geom("vstem", 1, 6, 3, 13, 10, 1, 64, 0, 0, 0, 2), S.Geom("astem", 2, 2, 1, 1, 640, 1, 64, 0, 0, 0, 1),
        S.Geom("v3x3", 0, 3, 1, 7, 6, 64, 64, 3, 3, 1, 2), S.Geom("v3x3s2", 0, 3, 1, 7, 6, 64, 128, 3, 3, 2, 2),
        S.Geom("vds", 0, 3, 1, 7, 6, 64, 128, 1, 1, 2, 2), S.Geom("a3s2", 0, 2, 1, 1, 21, 64, 128, 1, 3, 2, 1),
        S.Geom("a1", 0, 2, 1, 1, 21, 64, 64, 1, 3, 1, 1)]


@pytest.mark.parametrize("g", TINY, ids=lambda g: g.name)
@pytest.mark.parametrize("act,resid", [(True, False), (True, True), (False, False)])
def test_oracle_is_torchs_unit(g, act, resid):
    args, dy = _unit_inputs(g, resid)
    a = S.unit(*args, act, dy)
    b = S.torch_unit(*args, act, dy)
    for q in a:
        if a[q] is None:
            assert b[q] is None, q
        else:
            assert S.rel(a[q], b[q]) < 1e-12, (q, S.rel(a[q], b[q]))


@pytest.mark.parametrize("defect", list(S.DEFECTS))
def test_every_defect_changes_the_oracle(defect):
    hit = 0
    for g in TINY:
        for act, resid in ((True, True), (True, False)):
            if not S.applies(defect, g, act, resid):
                continue
            args, dy = _unit_inputs(g, resid, seed=1)
            a = S.unit(*args, act, dy, splits=3)
            b = S.unit(*args, act, dy, splits=3, defect=defect)
            worst = max(S.rel(b[q], a[q]) for q in a if a[q] is not None)
            assert worst > 1e-6, (g.name, defect, worst)      # float64 rounding is ~1e-15
            hit += 1
    assert hit > 0


def test_pool_by_winner_is_max_pool_when_the_winners_agree():
    gen = torch.Generator().manual_seed(3)
    x = torch.randn(2, 8, 3, 9, 12, generator=gen, dtype=torch.float64)          # (B, C, T, H, W): no ties
    xr = x.clone().requires_grad_(True)
    ref = torch.nn.functional.max_pool3d(xr, (1, 3, 3), (1, 2, 2), (0, 1, 1))
    dy = torch.randn(ref.shape, generator=gen, dtype=torch.float64)
    ref.backward(dy)
    # the window index of torch's winner
    xp = torch.nn.functional.pad(x, (1, 1, 1, 1), value=float("-inf"))
    Ho, Wo = ref.shape[-2:]
    cand = torch.stack([xp[..., a:a + 2 * Ho - 1:2, b:b + 2 * Wo - 1:2] for a in range(3) for b in range(3)])
    idx = (cand == ref.detach()[None]).to(torch.uint8).argmax(0)                  # (B, C, T, Ho, Wo)
    idx = idx.permute(0, 2, 3, 4, 1).reshape(-1, Ho, Wo, 8)
    xl = x.clone().requires_grad_(True)
    y = S.pool_by_winner(xl, idx)
    y.backward(dy)
    assert torch.equal(y.detach(), ref.detach()) and torch.equal(xl.grad, xr.grad)
