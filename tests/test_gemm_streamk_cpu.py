"""CPU check of the tensor-core GEMM's stream-K work list (csrc/gemm_schedule.cuh, compiled for the host from the same
header the kernel includes).  Stream-K gives every CTA a contiguous, equal share of a GEMM's (tile, k-block) steps;
a tile shared by several CTAs is finished by the last of them to arrive, which sums the pieces' fp32 partials in
piece order.  For every shape, operand width, tile width and SM count below:
  - every (tile, k-block) is computed exactly once;
  - each CTA's share is contiguous in step order and within one k-block of every other CTA's;
  - no tile has more pieces than there are partial planes (kMaxSplits), and a tile's pieces are numbered 0, 1, ...
    in k order with the same piece count;
  - under every arrival order of a tile's pieces, the counter protocol of gemm_tc_kernel elects exactly one finisher,
    leaves the counter at zero, and the finisher's sum is the same bits whatever the order.
The equal-slice split-K list gives the same piece descriptors (piece = K-slice, npieces = splits)."""
import ctypes as C
import itertools
import os
import random
import shutil
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SRC = os.path.join(HERE, "emu", "gemm_streamk_emu.cu")
OUT = os.path.join(HERE, "emu", "_build", "libgemm_streamk_emu.so")
DEPS = [SRC, os.path.join(ROOT, "auto_avsr_b200", "csrc", "gemm_schedule.cuh"),
        os.path.join(ROOT, "auto_avsr_b200", "csrc", "common.cuh")]
NVCC = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"

MS = (1, 100, 127, 128, 129, 1600, 2000, 3200)
NS = (8, 136, 768)
KS = (64, 768, 3072)
KE = {"tf32": 32, "f16": 64}        # K elements per 128-byte k-block
SMS = (132, 114, 78, 7, 1)


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(NVCC):
        pytest.skip("nvcc is needed to build the host replay")
    if not os.path.exists(OUT) or any(os.path.getmtime(d) > os.path.getmtime(OUT) for d in DEPS):
        os.makedirs(os.path.dirname(OUT), exist_ok=True)
        r = subprocess.run([NVCC, "-std=c++17", "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-shared", "-o", OUT,
                            SRC], capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
    so = C.CDLL(OUT)
    so.tc_emu_max_splits.restype = C.c_int
    so.tc_emu_sk_ctas.restype = C.c_int
    so.tc_emu_sk_ctas.argtypes = [C.c_int] * 3
    for fn, n in ((so.tc_emu_sk_walk, 4), (so.tc_emu_slice_walk, 5)):
        fn.restype = C.c_int
        fn.argtypes = [C.c_int] * n + [C.POINTER(C.c_int), C.c_int]
    return so


def walk(fn, *args):
    """rows {cta, j, tm, tn, kb0, kb1, piece, npieces} of a piece list"""
    cap = 1 << 16
    buf = (C.c_int * (8 * cap))()
    n = fn(*args, buf, cap)
    assert n < cap
    return np.frombuffer(buf, dtype=np.int32, count=8 * n).reshape(n, 8)


def check_pieces(rows, tiles_m, tiles_n, nkb, max_splits, ctx):
    """every (tile, k-block) once; a tile's pieces tile [0, nkb) in k order, numbered 0.. with one piece count"""
    by_tile = {}
    for cta, _, tm, tn, kb0, kb1, piece, npieces in rows.tolist():
        assert 0 <= tm < tiles_m and 0 <= tn < tiles_n and 0 <= kb0 < kb1 <= nkb, ctx
        by_tile.setdefault((tm, tn), []).append((kb0, kb1, piece, npieces, cta))
    assert len(by_tile) == tiles_m * tiles_n, ctx
    for tile, ps in by_tile.items():
        ps.sort()
        assert ps[0][0] == 0 and ps[-1][1] == nkb, (ctx, tile)
        assert all(a[1] == b[0] for a, b in zip(ps, ps[1:])), (ctx, tile)
        assert [p[2] for p in ps] == list(range(len(ps))), (ctx, tile)
        assert {p[3] for p in ps} == {len(ps)} and len(ps) <= max_splits, (ctx, tile)
    return by_tile


def test_streamk_covers_each_step_once_in_equal_contiguous_shares(lib):
    kmax = lib.tc_emu_max_splits()
    for M, N, K, op, bn, sms in itertools.product(MS, NS, KS, KE, (64, 128), SMS):
        tiles_m, tiles_n, nkb = -(-M // 128), -(-N // bn), K // KE[op]
        tiles = tiles_m * tiles_n
        ctas = lib.tc_emu_sk_ctas(sms, tiles, nkb)
        ctx = (M, N, K, op, bn, sms, ctas)
        assert 1 <= ctas <= min(sms, tiles * nkb), ctx
        rows = walk(lib.tc_emu_sk_walk, ctas, tiles_m, tiles_n, nkb)
        check_pieces(rows, tiles_m, tiles_n, nkb, kmax, ctx)
        # shares: CTA c's pieces are consecutive global steps (tile-major, n fastest), CTA c + 1 goes on from there
        nxt, share = 0, {}
        for cta, j, tm, tn, kb0, kb1, *_ in rows.tolist():
            g0 = (tm * tiles_n + tn) * nkb + kb0
            assert g0 == nxt, ctx
            nxt = g0 + (kb1 - kb0)
            share[cta] = share.get(cta, 0) + kb1 - kb0
        assert nxt == tiles * nkb and sorted(share) == list(range(ctas)), ctx
        assert max(share.values()) - min(share.values()) <= 1, ctx


def test_fewer_ctas_rather_than_more_pieces(lib):
    """the encoder's residual GEMMs at S2 fill every SM; at S1 (100 rows: 6 tiles) the w_2 GEMM takes fewer CTAs"""
    assert lib.tc_emu_sk_ctas(132, 13 * 6, 3072 // 64) == 132
    assert lib.tc_emu_sk_ctas(132, 13 * 6, 768 // 64) == 132
    assert lib.tc_emu_sk_ctas(132, 13 * 6, 3072 // 32) == 132
    assert lib.tc_emu_sk_ctas(132, 6, 3072 // 64) < 132


def test_equal_slice_split_k_is_the_same_piece_descriptor(lib):
    kmax = lib.tc_emu_max_splits()
    for M, N, nkb, splits in itertools.product((1, 129, 1600), (136, 768), (12, 48), (1, 2, 3, kmax)):
        tiles_m, tiles_n = -(-M // 128), -(-N // 128)
        rows = walk(lib.tc_emu_slice_walk, 132, tiles_m, tiles_n, nkb, splits)
        by_tile = check_pieces(rows, tiles_m, tiles_n, nkb, kmax, (M, N, nkb, splits))
        for ps in by_tile.values():
            assert [(p[0], p[1]) for p in ps] == [(s * nkb // splits, (s + 1) * nkb // splits) for s in range(splits)]


def finish(pieces, order, counters, planes, own):
    """the counter protocol of gemm_tc_kernel's fix-up for one tile, pieces arriving in `order`: each arrival
    publishes its plane, then atomicAdd; the one that sees npieces - 1 re-arms the counter and sums bias + planes in
    piece order, its own plane from its registers.  Returns [(finisher, sum)]."""
    done = []
    n = len(pieces)
    for p in order:
        planes[p] = own[p]
        old = counters[0]
        counters[0] += 1
        if old == n - 1:
            counters[0] = 0
            acc = np.float32(0.25)
            for q in range(n):
                acc = np.float32(acc + (own[p] if q == p else planes[q]))
            done.append((p, acc))
    return done


def test_counter_protocol_elects_one_finisher_whose_sum_ignores_arrival_order(lib):
    rnd = random.Random(3)
    tiles_seen = set()
    for M, N, K, op, sms in itertools.product(MS, NS, KS, KE, SMS):
        tiles_m, tiles_n, nkb = -(-M // 128), -(-N // 128), K // KE[op]
        ctas = lib.tc_emu_sk_ctas(sms, tiles_m * tiles_n, nkb)
        rows = walk(lib.tc_emu_sk_walk, ctas, tiles_m, tiles_n, nkb)
        for tile, ps in check_pieces(rows, tiles_m, tiles_n, nkb, lib.tc_emu_max_splits(), ()).items():
            n = len(ps)
            if n == 1 or n in tiles_seen and rnd.random() < 0.9:
                continue
            tiles_seen.add(n)
            own = [np.float32(rnd.uniform(-1, 1) * 10 ** rnd.randint(-3, 3)) for _ in range(n)]
            orders = list(itertools.permutations(range(n))) if n <= 5 else \
                [tuple(range(n)), tuple(reversed(range(n)))] + [tuple(rnd.sample(range(n), n)) for _ in range(200)]
            sums = set()
            counters = [0]
            for order in orders:
                done = finish(ps, order, counters, [None] * n, own)
                assert len(done) == 1 and counters[0] == 0 and done[0][0] == order[-1]
                sums.add(done[0][1].tobytes())
            assert len(sums) == 1
    assert max(tiles_seen) >= 3
