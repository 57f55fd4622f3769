"""The MSM bucket sort (cs_msm.cuh msm_sort: k_msm_bin_count, k_msm_bin_scan, k_msm_bin_scatter) against a Python
recoding of the same scalars.

count[] must equal the reference bucket counts, start[] their exclusive prefix, and every bucket must hold exactly the
reference's entries (table slot w * nbases + offset + i | sign); the order inside a bucket is free.  The cases cover
uniform scalars, every entry in one bucket, zero scalars, sparse and full infinity masks with an offset, Rep3 shares
read with stride 2, Montgomery and canonical input, windows 2 to 20 (17 and 20 split the buckets over several
shared-memory histograms), n = 1 and n not a multiple of the tile.  CPU: the emulated kernels; GPU: the same cases
on the device.
"""
import ctypes
import os
import random
import subprocess
import sys

import numpy as np
import pytest

from co_snarks_b200 import binding as B
from helpers import Conv

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SHIM = os.path.join(HERE, "emu", "sort_shim.cpp")
INCLUDES = ["-I", os.path.join(HERE, "emu"), "-I", os.path.join(ROOT, "co_snarks_b200", "csrc")]
SIGN = 0x80000000
R = Conv("bn254").r

# name: (window c, n, scalar kind, Montgomery input, Rep3 stride, infinity mask kind, offset)
CASES = {
    "uniform_c16": (16, 5000, "uniform", 0, 1, None, 0),
    "uniform_c8_mont": (8, 5000, "uniform", 1, 1, None, 0),
    "one_bucket_c16": (16, 5000, "one_bucket", 0, 1, None, 0),
    "one_bucket_c8_mont": (8, 700, "one_bucket", 1, 1, None, 0),
    "zero_scalars": (8, 300, "zero", 0, 1, None, 0),
    "sparse_mask_offset": (16, 4200, "uniform", 1, 1, "sparse", 3),
    "full_mask_offset": (8, 300, "uniform", 0, 1, "full", 2),
    "rep3_stride2_mont": (16, 4500, "uniform", 1, 2, None, 0),
    "window2": (2, 300, "uniform", 0, 1, None, 0),
    "window17_two_tiles": (17, 9000, "uniform", 0, 1, "sparse", 1),
    "window20": (20, 600, "uniform", 1, 1, None, 0),
    "n1_c16": (16, 1, "uniform", 0, 1, None, 0),
    "n1_c2_mont": (2, 1, "uniform", 1, 1, None, 0),
}


def _windows(c):
    return (254 + 1 + c - 1) // c


def _scalars(kind, n, c, rng):
    if kind == "zero":
        return [0] * n
    if kind == "one_bucket":
        # the same digit d in every window (no carries), so all W n entries go to bucket d
        W = _windows(c)
        d = max(1, (1 << (c - 1)) // 3)
        while d * sum(1 << (c * w) for w in range(W)) >= R:
            d -= 1
        assert d >= 1
        return [d * sum(1 << (c * w) for w in range(W))] * n
    out = [rng.randrange(R) for _ in range(n)]
    for k in range(0, n, 7):  # small scalars (many zero digits) and zeros among them
        out[k] = rng.randrange(1 << 12) if k % 2 else 0
    return out


def _recode(s, c, W):
    half, mask, carry, out = 1 << (c - 1), (1 << c) - 1, 0, []
    for w in range(W):
        d = ((s >> (w * c)) & mask) + carry
        if d > half:
            out.append(((1 << c) - d) | SIGN)
            carry = 1
        else:
            out.append(d)
            carry = 0
    return out


def _case(name):
    c, n, kind, mont, stride, mask_kind, offset = CASES[name]
    rng = random.Random(name)
    scal = _scalars(kind, n, c, rng)
    nbases = n + offset + 5
    inf = [False] * nbases
    if mask_kind == "sparse":
        inf = [rng.random() < 0.3 for _ in range(nbases)]
    elif mask_kind == "full":
        inf = [True] * nbases
    stored = [(s << 256) % R if mont else s for s in scal]
    rows = []
    for s in stored:
        rows.append(s)
        if stride == 2:
            rows.append(rng.randrange(R))  # the `b` component of a Rep3 share, which the sort must not read
    limbs = np.ascontiguousarray(B.ints_to_limbs(rows, 4)).view(np.uint32).reshape(n * stride, 8)
    words = None
    if mask_kind:
        words = np.zeros((nbases + 31) // 32, dtype=np.uint32)
        for i, f in enumerate(inf):
            if f:
                words[i >> 5] |= np.uint32(1 << (i & 31))
    # reference: bucket -> sorted entries
    W, nb1 = _windows(c), (1 << (c - 1)) + 1
    ref = {}
    for i, s in enumerate(scal):
        if inf[offset + i]:
            continue
        for w, d in enumerate(_recode(s, c, W)):
            b = d & ~SIGN
            if b:
                ref.setdefault(b, []).append((w * nbases + offset + i) | (d & SIGN))
    return dict(c=c, n=n, mont=mont, stride=stride, offset=offset, nbases=nbases, limbs=limbs, words=words, W=W,
                nb1=nb1, ref={b: sorted(v) for b, v in ref.items()}, kind=kind, mask=mask_kind)


def _run_and_check(lib, name):
    k = _case(name)
    nb1, W, n = k["nb1"], k["W"], k["n"]
    count = np.zeros(nb1, dtype=np.uint32)
    start = np.zeros(nb1 + 1, dtype=np.uint32)
    out = np.zeros(max(W * n, 1), dtype=np.uint32)
    p = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_uint32))  # noqa: E731
    rc = lib.bucket_sort(n, p(k["limbs"]), k["stride"], k["mont"], k["c"], k["nbases"], k["offset"],
                         p(k["words"]) if k["words"] is not None else None, p(count), p(start), p(out))
    assert rc == 0
    ref_count = np.zeros(nb1, dtype=np.uint64)
    for b, v in k["ref"].items():
        ref_count[b] = len(v)
    assert count.tolist() == ref_count.tolist(), "bucket counts differ from the reference recoding"
    assert start.tolist() == np.concatenate([[0], np.cumsum(ref_count)]).tolist(), "start is not the prefix of count"
    total = int(ref_count.sum())
    got = out[:total]
    for b in np.nonzero(ref_count)[0].tolist():
        assert sorted(got[start[b]:start[b + 1]].tolist()) == k["ref"][b], f"bucket {b} holds other entries"
    if k["kind"] == "one_bucket":
        assert np.count_nonzero(ref_count) == 1 and total == W * n
    if k["kind"] == "zero" or k["mask"] == "full":
        assert total == 0


@pytest.fixture(scope="module")
def emu_shim(tmp_path_factory):
    sys.path.insert(0, os.path.join(HERE, "emu"))
    import build_emu
    emu = build_emu.build()
    out = str(tmp_path_factory.mktemp("sort_shim") / "libsort_shim.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-DCS_EMU", "-DCS_ENABLE_BLS12_381", "-fPIC", "-shared", "-w"]
                          + INCLUDES + ["-o", out, SHIM, emu, "-Wl,-rpath," + os.path.dirname(emu)])
    return ctypes.CDLL(out)


@pytest.fixture(scope="module")
def gpu_shim(tmp_path_factory):
    from co_snarks_b200 import build as cuda_build
    out = str(tmp_path_factory.mktemp("sort_shim_gpu") / "libsort_shim.so")
    subprocess.check_call([cuda_build.NVCC] + cuda_build.GENCODE + ["-O3", "-std=c++17", "--expt-relaxed-constexpr",
                           "-DCS_ENABLE_BLS12_381", "-Xcompiler", "-fPIC", "-shared", "-x", "cu"] + INCLUDES
                          + ["-o", out, SHIM])
    return ctypes.CDLL(out)


@pytest.mark.parametrize("case", list(CASES))
def test_bucket_sort_emu(emu_shim, case):
    _run_and_check(emu_shim, case)


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_bucket_sort_gpu(gpu_shim, case):
    _run_and_check(gpu_shim, case)
