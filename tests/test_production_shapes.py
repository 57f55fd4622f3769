"""The NTT and the MSM against exact references at the shapes production runs.

NTT: a transform of 2^k runs in ceil(k / 10) passes (cs_ntt.cuh), so 2^10 / 2^11, 2^20 / 2^21 are the last and first
sizes of one, two and three passes; only the middle pass of three has tiles with both a high and a low offset.  At
each, every output equals oracle/c's plain radix-2 loop, on BN254 and BLS12-381, both directions each on its own input,
so no error can cancel in a round trip (2^22 with batch 2 and 2^24: test_gpu_fullsize.py).  The 3-pass witness map
checks the coset table the last iNTT pass applies in its store.

MSM: at n >= 2^15 the automatic window is 16 bits: 2^15 buckets, 32-entry slices, three fold levels and the multi-block
final sum.  The bases are k_i G (cs_fixed_base_mul), so the expected value of any MSM is (sum s_i k_i mod r) G: one
oracle scalar multiplication at any n.  The scalar and base distributions aim at the cases uniform scalars reach only
by chance: one bucket holding W n entries, equal / opposite / infinite partials in every fold, digits of exactly half
the window and carries through every window, and bases at infinity.

Every window cs_bases_upload accepts runs an MSM; wider ones are refused at upload.  Small copies of the MSM checks run
on the CPU emulation of the kernels (tests/emu)."""
import os
import random
import subprocess
import sys

import numpy as np
import pytest

from co_snarks_b200 import binding as B
import kernel_checks as K
from helpers import Conv
from oracle.ec import g1 as og1, g2 as og2
from oracle.fields import CURVES

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAX_WINDOW = 20  # widest window the MSM's bucket scan takes (cs_bases_upload refuses wider ones)


def msm_auto_window(n, scalar_bits):
    """Python statement of msm_auto_window (csrc/cs_msm.cuh): the window cs_bases_upload picks for n bases."""
    lg = n.bit_length() - 1
    c = 16 if lg >= 15 else max(lg - 4, 4)
    while c < 16:
        W = (scalar_bits + 1 + c - 1) // c
        if 2 * (scalar_bits + 1 - (W - 1) * c) >= c:
            break
        c += 1
    return c


def windows(cv, c):
    """number of c-bit windows of the signed recoding (msm_shape: the top window keeps <= c - 1 bits)"""
    return (cv.r.bit_length() + 1 + c - 1) // c


# ------------------------------------------------------------------------------------------ scalar distributions
def witness_like(cv, n, rng):
    """Groth16 witnesses: mostly 0 and 1 -- a quarter of all scalars land in bucket 1 of window 0."""
    out = []
    for _ in range(n):
        u = rng.random()
        out.append(0 if u < 0.45 else 1 if u < 0.70 else rng.randrange(2, 1 << 16) if u < 0.90 else rng.randrange(cv.r))
    for i in range(0, n, max(1, n // 7)):
        out[i] = cv.r - 1
    return out


def one_bucket(cv, n, c):
    """The same digit d in every c-bit window (no carries), so all W n entries go to bucket d.  At c = 16 that is
    d = 12345 in all W = 16 windows (12345 * 2^240 < r on both curves); narrower windows leave the top one empty."""
    d = min(12345, (1 << (c - 1)) - 1)
    W = windows(cv, c)
    v = d * sum(1 << (c * w) for w in range(W))
    if v >= cv.r:
        v = d * sum(1 << (c * w) for w in range(W - 1))
    assert c != 16 or v >> 240 == d
    return [v] * n


def recoding_edges(cv, n, c, rng):
    """Windows 0..W-2 all equal to half (digit +2^(c-1), the top bucket), or all equal to half + 1 (negative digits with a
    carry through every window into the top one), mixed with scalars below 2^c (window 0 only)."""
    W = windows(cv, c)
    half = 1 << (c - 1)
    rep = sum(1 << (c * w) for w in range(W - 1))
    pats = [half * rep, (half + 1) * rep, rep * (half - 1), half]
    assert all(p < cv.r for p in pats)
    out = []
    for i in range(n):
        k = i % 6
        out.append(pats[k] if k < 4 else rng.randrange(1 << c))
    rng.shuffle(out)
    return out


# ------------------------------------------------------------------------------------------ known-discrete-log MSM
def dlog_bases(ctx, cv, group, ks):
    """Points k_i G for the ints ks (0 -> the point at infinity), each distinct k multiplied once on the device."""
    C_ = CURVES["bn254" if cv.id == B.CS_BN254 else "bls12_381"]
    gen = (cv.g1 if group == 0 else cv.g2)([C_.g1 if group == 0 else C_.g2])[0]
    uniq = sorted(set(ks))
    pos = {k: i for i, k in enumerate(uniq)}
    pts = ctx.fixed_base_mul(cv.id, group, gen, B.ints_to_limbs(uniq, 4), montgomery=False)
    return np.ascontiguousarray(pts[np.array([pos[k] for k in ks], dtype=np.int64)])


def expected(cv, group, ks, ss):
    C_ = CURVES["bn254" if cv.id == B.CS_BN254 else "bls12_381"]
    G = og1(C_) if group == 0 else og2(C_)
    return G.mul(C_.g1 if group == 0 else C_.g2, sum(s * k for s, k in zip(ss, ks)) % cv.r)


def run_msm(ctx, cv, group, bases, ks, ss, what):
    """The MSM with Montgomery and with canonical scalars against (sum s_i k_i) G; the infinity flag must agree."""
    exp = expected(cv, group, ks, ss)
    to_pt = cv.pt1 if group == 0 else cv.pt2
    for mont in (True, False):
        out, inf = ctx.msm(bases, cv.fr(ss) if mont else cv.fr_canonical(ss), montgomery=mont)
        assert to_pt(out) == exp, (what, "montgomery" if mont else "canonical")
        assert inf == (exp is None), (what, "infinity flag")


def check_msm_distributions(ctx, curve, group, n, window_bits=0, seed=1):
    """The distributions of the module docstring over three base sets: random k_i with some at infinity, one base
    repeated (every slice partial of a bucket is the same point, so the folds double), and k, r - k alternating (the
    folds meet equal and opposite partials and partials at infinity; the result is infinity)."""
    cv = Conv(curve)
    rng = random.Random(seed)
    c = window_bits or msm_auto_window(n, cv.r.bit_length())
    ks = [rng.randrange(1, cv.r) for _ in range(n)]
    for i in range(3, n, 17):
        ks[i] = 0
    bases = ctx.bases_upload(cv.id, group, dlog_bases(ctx, cv, group, ks), window_bits)
    run_msm(ctx, cv, group, bases, ks, witness_like(cv, n, rng), "witness-like")
    run_msm(ctx, cv, group, bases, ks, one_bucket(cv, n, c), "one bucket")
    run_msm(ctx, cv, group, bases, ks, recoding_edges(cv, n, c, rng), "recoding edges")
    run_msm(ctx, cv, group, bases, ks, [rng.randrange(cv.r) for _ in range(n)], "uniform")
    bases.free()
    k0 = rng.randrange(1, cv.r)
    same = [k0] * n
    bases = ctx.bases_upload(cv.id, group, dlog_bases(ctx, cv, group, same), window_bits)
    run_msm(ctx, cv, group, bases, same, [rng.randrange(cv.r)] * n, "equal partials")
    run_msm(ctx, cv, group, bases, same, one_bucket(cv, n, c), "equal partials, one bucket")
    bases.free()
    alt = [k0 if i % 2 == 0 else cv.r - k0 for i in range(n & ~1)]
    bases = ctx.bases_upload(cv.id, group, dlog_bases(ctx, cv, group, alt), window_bits)
    run_msm(ctx, cv, group, bases, alt, [rng.randrange(cv.r)] * len(alt), "cancelling partials")
    run_msm(ctx, cv, group, bases, alt, one_bucket(cv, len(alt), c), "cancelling partials, one bucket")
    bases.free()


def check_dlog_msm(ctx, curve, group, n, window_bits=0, seed=2):
    """Uniform scalars and uniform k_i at the given window (0 = automatic)."""
    cv = Conv(curve)
    rng = random.Random(seed)
    ks = [rng.randrange(cv.r) for _ in range(n)]
    bases = ctx.bases_upload(cv.id, group, dlog_bases(ctx, cv, group, ks), window_bits)
    run_msm(ctx, cv, group, bases, ks, [rng.randrange(cv.r) for _ in range(n)], "uniform")
    run_msm(ctx, cv, group, bases, ks, witness_like(cv, n, rng), "witness-like")
    bases.free()


def check_window_sweep(ctx, curve="bn254", n=64, seed=3):
    """Every window cs_bases_upload accepts, 2..20, against the oracle's MSM on the same points."""
    cv = Conv(curve)
    C_ = CURVES[curve]
    G = og1(C_)
    pts, sc = K._edge_case_inputs(G, C_.g1, n, cv.r, random.Random(seed))
    exp = G.msm(pts, sc)
    arr = cv.g1(pts)
    for wb in range(2, MAX_WINDOW + 1):
        bases = ctx.bases_upload(cv.id, 0, arr, wb)
        out, inf = ctx.msm(bases, cv.fr(sc))
        assert cv.pt1(out) == exp and inf == (exp is None), ("window", wb)
        out, _ = ctx.msm(bases, cv.fr_canonical(sc[1:]), offset=1, montgomery=False)
        assert cv.pt1(out) == G.msm(pts[1:], sc[1:]), ("window", wb, "offset 1")
        bases.free()


def check_window_rejected(ctx):
    """Windows the bucket scan cannot take fail at upload, and so does a Groth16 key built with one."""
    from helpers import golden_groth16, make_key
    cv = Conv("bn254")
    arr = cv.g1([CURVES["bn254"].g1] * 8)
    for wb in (MAX_WINDOW + 1, MAX_WINDOW + 2, 32, 1, -1):
        with pytest.raises(B.CsError, match="window_bits"):
            ctx.bases_upload(cv.id, 0, arr, wb)
    z, m, _, _ = golden_groth16("multiplier2")
    with pytest.raises(B.CsError, match="window_bits"):
        make_key(ctx, cv, z, m, window_bits=MAX_WINDOW + 1)
    make_key(ctx, cv, z, m, window_bits=MAX_WINDOW).free()


# ------------------------------------------------------------------------------------------ CPU emulation
def test_msm_auto_window_statement():
    """The Python statement above picks the documented windows (16 bits from 2^15 bases on)."""
    for bits in (254, 255):
        assert [msm_auto_window(1 << lg, bits) for lg in (15, 16, 20, 24)] == [16] * 4
        assert all(4 <= msm_auto_window(1 << lg, bits) <= 16 for lg in range(0, 15))


def test_emu_ntt_one_and_two_pass_against_oracle_c(emu_ctx):
    for curve in ("bn254", "bls12_381"):
        for lg, batch in ((10, 1), (10, 2), (11, 1), (11, 2)):
            K.check_ntt_against_oracle_c(emu_ctx, curve, lg, batch)


def test_emu_fixed_base_mul_bls12_381(emu_ctx):
    K.check_fixed_base_mul(emu_ctx, n=24, curve="bls12_381")


def test_emu_msm_every_accepted_window(emu_ctx):
    check_window_sweep(emu_ctx)


def test_emu_msm_window_above_scan_rejected(emu_ctx):
    check_window_rejected(emu_ctx)


@pytest.mark.parametrize("curve,group,n", [("bn254", 0, 600), ("bn254", 1, 150), ("bls12_381", 0, 300),
                                           ("bls12_381", 1, 80)])
def test_emu_msm_distributions_16bit_window(emu_ctx, curve, group, n):
    """The production window forced on a small n: 2^15 buckets, the multi-block final sum, the same distributions."""
    check_msm_distributions(emu_ctx, curve, group, n, window_bits=16)


def test_emu_msm_distributions_auto_window(emu_ctx):
    check_msm_distributions(emu_ctx, "bn254", 0, 700)


# ------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("lg,batch", [(10, 1), (11, 1), (11, 2), (20, 1), (21, 1), (21, 2)])
def test_ntt_bn254_matches_oracle_c(gpu_ctx, lg, batch):
    """2^22 with batch 2 and 2^24: test_gpu_fullsize.py::test_ntt_plonk_sizes_roundtrip."""
    K.check_ntt_against_oracle_c(gpu_ctx, "bn254", lg, batch)


@pytest.mark.gpu
@pytest.mark.parametrize("lg,batch", [(11, 1), (11, 2), (16, 1), (20, 1), (21, 1), (22, 2)])
def test_ntt_bls12_381_matches_oracle_c(gpu_ctx, lg, batch):
    K.check_ntt_against_oracle_c(gpu_ctx, "bls12_381", lg, batch)


@pytest.mark.gpu
def test_ntt_tma_pass_matches_oracle_c_subprocess():
    """The opt-in TMA-staged radix-8 pass (CS_NTT_V2=1) at 2^20 and 2^22 with batch 2.  Separate process: the switch is
    read once per process."""
    code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r);"
            "from co_snarks_b200 import binding as B; import kernel_checks as K; ctx = B.Context(0);"
            "K.check_ntt_against_oracle_c(ctx, 'bn254', 20, 1); K.check_ntt_against_oracle_c(ctx, 'bn254', 22, 2);"
            "K.check_ntt_against_oracle_c(ctx, 'bls12_381', 21, 1); print('ok')" % (ROOT, os.path.join(ROOT, "tests")))
    env = dict(os.environ, CS_NTT_V2="1")
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and "ok" in out.stdout, out.stdout + out.stderr


@pytest.mark.gpu
def test_groth16_witness_map_three_pass_coset_matches_oracle_c(gpu_ctx):
    """The witness map at 2^21 (three-pass NTTs; the coset table is applied by the last iNTT pass's fused store) equals
    oracle/c's on every output.  A random one-entry-per-row R1CS over 8 variables: only the domain size matters here,
    so the query points are all at infinity."""
    from oracle.c import run as OC
    cv = Conv("bn254")
    lg, ni, nv = 21, 2, 8
    n = 1 << lg
    nc = n - ni
    rng = np.random.Generator(np.random.PCG64(21))

    def csr():
        return (np.arange(nc + 1, dtype=np.uint32), rng.integers(0, nv, size=nc, dtype=np.uint32),
                K.rand_fr_limbs(nc, int(rng.integers(1 << 30))))
    mats = dict(num_constraints=nc, num_instance_variables=ni, num_witness_variables=nv - ni, a=csr(), b=csr())
    g1 = lambda k: np.zeros((k, 8), dtype=np.uint64)
    g2 = lambda k: np.zeros((k, 16), dtype=np.uint64)
    pts = dict(alpha_g1=g1(1), beta_g1=g1(1), beta_g2=g2(1), delta_g1=g1(1), delta_g2=g2(1), a_query=g1(nv),
               b_g1_query=g1(nv), b_g2_query=g2(nv), l_query=g1(nv - ni), h_query=g1(n))
    pub, wit = K.rand_fr_limbs(ni, 1), K.rand_fr_limbs(nv - ni, 2)
    pk = B.Groth16Key(gpu_ctx, cv.id, mats, pts)
    assert pk.domain_size() == n
    h = pk.witness_map(pub, wit)
    pk.free()
    desc, keep = OC.key_desc(mats, pts)
    exp = OC.witness_map(desc, 0, 0, pub, wit)
    del keep
    assert np.array_equal(h, exp), "%d of %d outputs differ" % (int((h != exp).any(axis=1).sum()), n)


@pytest.mark.gpu
def test_fixed_base_mul_bls12_381(gpu_ctx):
    K.check_fixed_base_mul(gpu_ctx, n=40, curve="bls12_381")


@pytest.mark.gpu
@pytest.mark.parametrize("curve,group,logn", [("bls12_381", 0, 16), ("bls12_381", 0, 20), ("bls12_381", 1, 16)])
def test_msm_bls12_381_production_window(gpu_ctx, curve, group, logn):
    assert msm_auto_window(1 << logn, Conv(curve).r.bit_length()) == 16
    check_dlog_msm(gpu_ctx, curve, group, 1 << logn)


@pytest.mark.gpu
@pytest.mark.parametrize("curve,group,logn", [("bn254", 0, 20), ("bn254", 1, 16), ("bls12_381", 0, 16)])
def test_msm_distributions_production_window(gpu_ctx, curve, group, logn):
    assert msm_auto_window(1 << logn, Conv(curve).r.bit_length()) == 16
    check_msm_distributions(gpu_ctx, curve, group, 1 << logn)


@pytest.mark.gpu
def test_msm_every_accepted_window(gpu_ctx):
    check_window_sweep(gpu_ctx)


@pytest.mark.gpu
@pytest.mark.parametrize("window_bits", [18, 20])
def test_msm_wide_window_2p16(gpu_ctx, window_bits):
    """Windows of 18 and 20 bits take the 64-entry slice path."""
    check_dlog_msm(gpu_ctx, "bn254", 0, 1 << 16, window_bits=window_bits)


@pytest.mark.gpu
def test_msm_window_above_scan_rejected(gpu_ctx):
    check_window_rejected(gpu_ctx)
