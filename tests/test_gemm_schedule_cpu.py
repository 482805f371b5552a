"""CPU check of the tensor-core GEMM's persistent work list (csrc/gemm_schedule.cuh, compiled for the host from the same
header the kernel includes): for every cluster shape, every output tile (and K-slice) is computed exactly once, and
all CTAs of a cluster walk the same number of items, item by item in the same cluster tile.  That is what keeps every
multicast load a CTA waits for matched by its peers' loads, so the GPU kernel cannot wait on a load nobody issues."""
import ctypes as C
import os
import shutil
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SRC = os.path.join(HERE, "emu", "gemm_schedule_emu.cu")
OUT = os.path.join(HERE, "emu", "_build", "libgemm_schedule_emu.so")
DEPS = [SRC, os.path.join(ROOT, "auto_avsr_b200", "csrc", "gemm_schedule.cuh"),
        os.path.join(ROOT, "auto_avsr_b200", "csrc", "common.cuh")]
NVCC = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"

CLUSTERS = [(1, 1), (2, 1), (1, 2), (2, 2)]
SMS = 132
# (M, N, BN): the encoder at S1/S2/S4 lengths, the head (ctc_lo N = 5120), the decoder (M <= 40), training dgrad /
# wgrad shapes, and the edges of tests/test_zz_gpu_gemm_cluster.py
SHAPES = [(m, n, bn) for m in (1, 64, 127, 128, 129, 1600, 1601, 3200) for n in (8, 72, 136, 768, 3072) for bn in (64, 128)]
SHAPES += [(1600, 2304, 128), (1600, 1536, 128), (799, 768, 128), (1600, 5120, 128), (40, 768, 64), (40, 5120, 128),
           (768, 3072, 128), (3072, 768, 128), (768, 768, 64)]


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
    so.tc_emu_items.restype = C.c_int
    so.tc_emu_items.argtypes = [C.c_int] * 5
    so.tc_emu_work.restype = None
    so.tc_emu_work.argtypes = [C.c_int] * 6 + [C.POINTER(C.c_int)]
    return so


def walk(lib, tiles_m, tiles_n, splits, cm, cn):
    """{cta: [(tm, tn, split, valid), ...]} of a persistent grid of SMS // (cm * cn) clusters."""
    cs = cm * cn
    clusters = SMS // cs
    items = lib.tc_emu_items(tiles_m, tiles_n, splits, cm, cn)
    buf = (C.c_int * 4)()
    seq = {}
    for cid in range(min(items, clusters)):
        for r in range(cs):
            out = []
            for item in range(cid, items, clusters):
                lib.tc_emu_work(item, r, tiles_m, tiles_n, cm, cn, buf)
                out.append(tuple(buf))
            seq[(cid, r)] = out
    return seq


@pytest.mark.parametrize("cm,cn", CLUSTERS)
def test_work_list_covers_each_tile_once(lib, cm, cn):
    for M, N, bn in SHAPES:
        tiles_m, tiles_n = -(-M // 128), -(-N // bn)
        for splits in ((1, 3) if cm * cn == 1 else (1,)):
            seq = walk(lib, tiles_m, tiles_n, splits, cm, cn)
            done = [w[:3] for s in seq.values() for w in s if w[3]]
            want = [(tm, tn, sp) for tm in range(tiles_m) for tn in range(tiles_n) for sp in range(splits)]
            assert sorted(done) == want, (M, N, bn, cm, cn, splits)
            for s in seq.values():
                for tm, tn, sp, valid in s:
                    assert bool(valid) == (tm < tiles_m and tn < tiles_n)
            # the CTAs of a cluster: same item count, and at each step tiles of one cluster tile in rank order
            for cid in {c for c, _ in seq}:
                peers = [seq[(cid, r)] for r in range(cm * cn)]
                assert len({len(p) for p in peers}) == 1, (M, N, bn, cm, cn, cid)
                for step in zip(*peers):
                    base_m, base_n = step[0][0], step[0][1]
                    assert base_m % cm == 0 and base_n % cn == 0
                    for r, (tm, tn, sp, _) in enumerate(step):
                        assert (tm, tn, sp) == (base_m + r % cm, base_n + r // cm, step[0][2])
