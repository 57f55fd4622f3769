"""Lazy-reduced Fp2 arithmetic (cs_field.cuh / cs_curve.cuh) against Python integers, on BN254 and BLS12-381.

The Fp2 product and a b - c d sum unreduced 2N-word products with offsets of p^2 and 2 p^2 and reduce once per
coefficient; this checks them, and the unreduced product and the reduction they are built from, on random operands
and on the operands at the ends of each bound (0, 1, p - 1, p - 2, coefficients whose unreduced sum is 2p - 2).  A
too-small offset wraps the sum and a too-large one breaks the reduction's input bound, so either shows up here.
The exact device algorithms run on the CPU through the emulated carry chain (tests/emu/fp2_shim.cpp)."""
import ctypes
import itertools
import os
import random
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

CURVES = {
    "bn254": (21888242871839275222246405745257275088696311157297823662689037894645226208583, 8),
    "bls381": (int("1a0111ea397fe69a4b1ba7b6434bacd764774b84f38512bf6730d2a0f6b0f6241eabfffeb153ffffb9feffffffffaaab", 16), 12),
}


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("fp2_shim") / "libfp2_shim.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-DCS_EMU", "-DCS_ENABLE_BLS12_381", "-fPIC", "-shared", "-w",
                           "-I", os.path.join(HERE, "emu"), "-I", os.path.join(ROOT, "co_snarks_b200", "csrc"),
                           "-o", out, os.path.join(HERE, "emu", "fp2_shim.cpp")])
    return ctypes.CDLL(out)


def pack(vals, words):
    return np.frombuffer(b"".join(v.to_bytes(4 * words, "little") for v in vals), dtype=np.uint32).copy()


def unpack(arr, words):
    b = arr.tobytes()
    return [int.from_bytes(b[4 * words * k:4 * words * (k + 1)], "little") for k in range(len(arr) // words)]


def ptr(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_uint32))


def call(lib, name, words_out, n, *args):
    out = np.zeros(n * words_out, dtype=np.uint32)
    getattr(lib, name)(ctypes.c_int(n), *[ptr(a) for a in args], ptr(out))
    return out


def fp2_pack(pairs, N):
    return pack([c for pr in pairs for c in pr], N)


def fp2_unpack(arr, N):
    v = unpack(arr, N)
    return list(zip(v[0::2], v[1::2]))


def edges(p):
    return [0, 1, p - 1, p - 2, (p - 1) // 2]


def fp2_operands(p, rng, n_random):
    e = edges(p)
    ops = list(itertools.product(e, e))  # includes (p - 1, p - 1): the unreduced sum 2p - 2
    ops += [(rng.randrange(p), rng.randrange(p)) for _ in range(n_random)]
    return ops


@pytest.mark.parametrize("curve", sorted(CURVES))
def test_mul_wide_and_redc(shim, curve):
    p, N = CURVES[curve]
    R = 1 << (32 * N)
    rinv = pow(R, -1, p)
    rng = random.Random(11)
    amax = (R >> 1) - 1  # mul_wide's bound on its first operand; the second is any N-word value
    a = [0, 1, p - 1, 2 * p - 2, amax, amax] + [rng.randrange(R >> 1) for _ in range(300)]
    b = [0, p - 1, 2 * p - 2, R - 1, 1, 2 * p - 2] + [rng.randrange(R) for _ in range(300)]
    got = unpack(call(shim, curve + "_mul_wide", 2 * N, len(a), pack(a, N), pack(b, N)), 2 * N)
    assert got == [x * y for x, y in zip(a, b)]
    # the reduction's whole input range: t < p R
    t = [0, 1, p - 1, p, p * p, 4 * (p - 1) ** 2, p * R - 1, R - 1, (p - 1) * R + R - 1] + \
        [rng.randrange(p * R) for _ in range(500)]
    got = unpack(call(shim, curve + "_redc", N, len(t), pack(t, 2 * N)), N)
    assert got == [x * rinv % p for x in t]


@pytest.mark.parametrize("curve", sorted(CURVES))
def test_fp2_mul(shim, curve):
    p, N = CURVES[curve]
    rinv = pow(1 << (32 * N), -1, p)
    rng = random.Random(12)
    ops = fp2_operands(p, rng, 100)
    pairs = list(itertools.product(ops[:25], ops[:25])) + [(rng.choice(ops), rng.choice(ops)) for _ in range(600)]
    a = [x for x, _ in pairs]
    b = [y for _, y in pairs]
    got = fp2_unpack(call(shim, curve + "_fp2_mul", 2 * N, len(pairs), fp2_pack(a, N), fp2_pack(b, N)), N)
    exp = [((x0 * y0 - x1 * y1) * rinv % p, (x0 * y1 + x1 * y0) * rinv % p) for (x0, x1), (y0, y1) in pairs]
    assert got == exp


@pytest.mark.parametrize("curve", sorted(CURVES))
def test_fp2_mul_sub(shim, curve):
    p, N = CURVES[curve]
    rinv = pow(1 << (32 * N), -1, p)
    rng = random.Random(13)
    ops = fp2_operands(p, rng, 100)
    m = p - 1
    # the ends of both coefficient bounds: a b - c d with one product at zero and the other at its largest
    quads = [((m, m), (m, m), (m, m), (m, m)),
             ((0, m), (0, m), (m, 0), (m, 0)),   # coefficient 0 at -2 (p-1)^2
             ((m, 0), (m, 0), (0, m), (0, m)),   # coefficient 0 at +2 (p-1)^2
             ((0, 0), (0, 0), (m, m), (m, m)),   # coefficient 1 at -2 (p-1)^2
             ((m, m), (m, m), (0, 0), (0, 0))]   # coefficient 1 at +2 (p-1)^2
    e = ops[:25]
    quads += [(rng.choice(e), rng.choice(e), rng.choice(e), rng.choice(e)) for _ in range(2000)]
    quads += [tuple(rng.choice(ops) for _ in range(4)) for _ in range(500)]
    cols = [fp2_pack([q[i] for q in quads], N) for i in range(4)]
    got = fp2_unpack(call(shim, curve + "_fp2_mul_sub", 2 * N, len(quads), *cols), N)

    def mul(x, y):
        return (x[0] * y[0] - x[1] * y[1], x[0] * y[1] + x[1] * y[0])

    exp = []
    for a, b, c, d in quads:
        u, w = mul(a, b), mul(c, d)
        exp.append(((u[0] - w[0]) * rinv % p, (u[1] - w[1]) * rinv % p))
    assert got == exp
