"""MSM tables with one row per k windows: what a base set or Groth16 key keeps when its full tables do not fit.

cs_bases_upload keeps T = ceil(W / k) rows, row j = 2^(c k j) P_i, and an MSM puts window w in row w / k and bucket group
w % k, then combines the k group sums by Horner's rule.  k is the smallest whose bytes fit the table budget (what the
device has free, capped by cs_ctx_set_table_budget); k = 1 is the full table.  The results must not depend on k, bit
for bit.

CPU (emulation build): every k in {1, 2, 3, W - 1, W} through a shim that uploads with an exact k (the budget reaches
only the smallest k of each row count), against the known discrete log of every base and against k = 1; Groth16 golden
proofs through keys with k = 2 and with one row, made by the same shim; the budget's semantics.
GPU: compact tables at 2^16 and 2^20 against full ones, the trapdoor references at 2^20 through compact keys (plain, Rep3
with three party threads on one GPU, Shamir(3, 1)), and a 2^24 BN254 key, which does not fit an 80 GB H100 with full
tables, proven and checked against oracle/c.
"""
import ctypes
import os
import random
import subprocess
import sys
import threading

import numpy as np
import pytest

from co_snarks_b200 import binding as B
from helpers import Conv, golden_groth16, ih, make_key
from oracle import groth16 as OG
from oracle.ec import g1 as og1, g2 as og2
from oracle.fields import CURVES
from workloads.random_groth16 import forced_key, rand_fr_limbs, random_key

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SHIM = os.path.join(HERE, "emu", "rows_shim.cpp")
ERR_LIMIT = -3


def windows(cv, c):
    return (cv.r.bit_length() + 1 + c - 1) // c


def auto_window(n, bits):
    """msm_auto_window (csrc/cs_msm.cuh)"""
    lg = n.bit_length() - 1
    c = 16 if lg >= 15 else max(lg - 4, 4)
    while c < 16:
        W = (bits + 1 + c - 1) // c
        if 2 * (bits + 1 - (W - 1) * c) >= c:
            break
        c += 1
    return c


@pytest.fixture
def budget_reset():
    """contexts whose table budget a test changes; reset to automatic afterwards"""
    ctxs = []
    yield ctxs.append
    for c in ctxs:
        c.set_table_budget(0)


# ------------------------------------------------------------------------------------------------ inputs
def dlog_bases(ctx, cv, group, ks):
    cd = CURVES["bn254" if cv.id == B.CS_BN254 else "bls12_381"]
    gen = (cv.g1 if group == 0 else cv.g2)([cd.g1 if group == 0 else cd.g2])[0]
    uniq = sorted(set(ks))
    pos = {k: i for i, k in enumerate(uniq)}
    pts = ctx.fixed_base_mul(cv.id, group, gen, B.ints_to_limbs(uniq, 4), montgomery=False)
    return np.ascontiguousarray(pts[np.array([pos[k] for k in ks], dtype=np.int64)])


def expected(cv, group, ks, ss):
    cd = CURVES["bn254" if cv.id == B.CS_BN254 else "bls12_381"]
    G = og1(cd) if group == 0 else og2(cd)
    return G.mul(cd.g1 if group == 0 else cd.g2, sum(s * k for s, k in zip(ss, ks)) % cv.r)


def base_dlogs(cv, n, rng):
    """random discrete logs with bases at infinity (0), duplicated bases and negated bases"""
    ks = [rng.randrange(1, cv.r) for _ in range(n)]
    for i in range(n):
        if i % 11 == 3:
            ks[i] = 0
        elif i % 13 == 5:
            ks[i] = ks[1 % n]
        elif i % 17 == 7:
            ks[i] = cv.r - ks[2 % n]
    return ks


def scalar_sets(cv, n, rng):
    """edge scalars (0, 1, r - 1, small and random mixed) and all-equal scalars (one bucket per window)"""
    edge = [(0, 1, cv.r - 1, rng.randrange(1 << 20), rng.randrange(cv.r))[i % 5] for i in range(n)]
    return [edge, [rng.randrange(cv.r)] * n]


# ------------------------------------------------------------------------------------------------ CPU emulation
@pytest.fixture(scope="module")
def rows_shim(emu_ctx, tmp_path_factory):
    sys.path.insert(0, os.path.join(HERE, "emu"))
    import build_emu
    emu = build_emu.build()
    out = str(tmp_path_factory.mktemp("rows_shim") / "librows_shim.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-DCS_EMU", "-DCS_ENABLE_BLS12_381", "-fPIC", "-shared", "-w",
                           "-I", os.path.join(HERE, "emu"), "-I", os.path.join(ROOT, "co_snarks_b200", "csrc"),
                           "-o", out, SHIM, emu, "-Wl,-rpath," + os.path.dirname(emu)])
    lib = ctypes.CDLL(out)
    lib.bases_upload_rows.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t,
                                      ctypes.c_int, ctypes.c_uint, ctypes.POINTER(ctypes.c_void_p)]
    lib.bases_upload_rows.restype = ctypes.c_int
    lib.groth16_pk_create_rows.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint, ctypes.c_void_p]
    lib.groth16_pk_create_rows.restype = ctypes.c_int
    lib.heap_bytes_in_use.restype = ctypes.c_size_t
    return lib


class _KeyRowsCtx:
    """The emulation context, with cs_groth16_pk_create replaced by the shim's creation at exactly k windows per row,
    so that B.Groth16Key builds its descriptor as usual."""

    def __init__(self, ctx, shim, k):
        self._ctx, self._shim, self._k = ctx, shim, k
        self.lib = self
        self.h, self._check = ctx.h, ctx._check

    def cs_groth16_pk_create(self, ctx_h, desc, out):
        return self._shim.groth16_pk_create_rows(ctx_h, desc, self._k, out)

    def __getattr__(self, name):
        return getattr(self._ctx.lib, name)


def key_rows(shim, ctx, cv, z, m, k):
    return make_key(_KeyRowsCtx(ctx, shim, k), cv, z, m)


def upload_rows(shim, ctx, cv, group, pts, wb, k):
    h = ctypes.c_void_p()
    ctx._check(shim.bases_upload_rows(ctx.h, cv.id, group, pts.ctypes.data_as(ctypes.c_void_p), pts.shape[0], wb, k,
                                      ctypes.byref(h)))
    b = B.Bases(ctx, h, cv.id, group)
    info = b.info()
    W = info["windows"]
    assert info["table_rows"] == (W + k - 1) // k
    return b


def ks_of(W):
    return sorted({1, 2, 3, W - 1, W})


# (curve, group, n, windows): every window at small n; 16-bit windows (2^15 buckets per group) at n = 4096 on G1
MSM_CASES = [(c, g, n, wbs) for c in ("bn254", "bls12_381") for g in (0, 1) for n, wbs in ((1, (0, 5)), (37, (0, 5, 7)),
                                                                                            (300, (0, 7, 16)))]
MSM_CASES += [("bn254", 0, 4096, (0, 16)), ("bls12_381", 0, 4096, (0,)), ("bn254", 1, 4096, (0,))]


@pytest.mark.parametrize("curve,group,n,wbs", MSM_CASES, ids=lambda v: str(v).replace(" ", ""))
def test_msm_every_k_emu(emu_ctx, rows_shim, curve, group, n, wbs):
    """cs_msm and cs_msm_rep3_shares with k in {1, 2, 3, W - 1, W}: equal to (sum s_i k_i) G and to k = 1 bit for bit."""
    cv = Conv(curve)
    rng = random.Random(hash((curve, group, n)) & 0xffff)
    ks = base_dlogs(cv, n, rng)
    pts = dlog_bases(emu_ctx, cv, group, ks)
    sets = scalar_sets(cv, n, rng)
    shares = [rng.randrange(cv.r) for _ in range(2 * n)]
    for wb in wbs:
        W = windows(cv, wb or auto_window(n, cv.r.bit_length()))
        full = None
        for k in ks_of(W):
            b = upload_rows(rows_shim, emu_ctx, cv, group, pts, wb, k)
            got = [emu_ctx.msm(b, cv.fr(ss))[0] for ss in sets]
            got.append(emu_ctx.msm(b, cv.fr_canonical(sets[0][1:]), offset=1, montgomery=False)[0])
            got += list(emu_ctx.msm_rep3_shares(b, cv.fr(shares).reshape(n, 8)))
            b.free()
            if full is None:
                full = got
                to_pt = cv.pt1 if group == 0 else cv.pt2
                for ss, out in zip(sets, got):
                    assert to_pt(out) == expected(cv, group, ks, ss), (wb, k)
                assert to_pt(got[2]) == expected(cv, group, ks[1:], sets[0][1:]), (wb, k, "offset 1")
                assert to_pt(got[3]) == expected(cv, group, ks, shares[0::2]), (wb, k, "rep3 a")
                assert to_pt(got[4]) == expected(cv, group, ks, shares[1::2]), (wb, k, "rep3 b")
            else:
                assert all(np.array_equal(a, x) for a, x in zip(got, full)), ("k", k, "window", wb)


def test_msm_every_k_slice64_emu(emu_ctx, rows_shim, monkeypatch):
    """The 64-entry slice path (CS_MSM_SLICE=64) with every k."""
    monkeypatch.setenv("CS_MSM_SLICE", "64")
    cv = Conv("bn254")
    rng = random.Random(64)
    n = 600
    ks = base_dlogs(cv, n, rng)
    pts = dlog_bases(emu_ctx, cv, 0, ks)
    ss = [rng.randrange(cv.r)] * n  # all equal: long buckets
    for k in ks_of(windows(cv, 7)):
        b = upload_rows(rows_shim, emu_ctx, cv, 0, pts, 7, k)
        assert cv.pt1(emu_ctx.msm(b, cv.fr(ss))[0]) == expected(cv, 0, ks, ss), k
        b.free()


GOLDEN = [("bn254", "multiplier2"), ("bn254", "poseidon"), ("bls12_381", "multiplier2"), ("bls12_381", "poseidon")]


@pytest.mark.parametrize("curve,name", GOLDEN)
def test_groth16_golden_compact_keys_emu(emu_ctx, rows_shim, curve, name):
    """Golden fixtures through keys with k = 2 and with one table row: the golden proofs, and the Rep3 local phase and
    cs_groth16_shamir_local equal to those of the full key."""
    cv = Conv(curve)
    z, m, w, g = golden_groth16(name, curve)
    ni = m["num_instance_variables"]
    pub, wit = cv.fr(w[:ni]), cv.fr(w[ni:])
    rng = random.Random(7)
    wsh = OG.share_rep3(w[ni:], cv.r, rng)
    sh0 = cv.fr([x for ab in wsh[0] for x in ab]).reshape(-1, 8)
    n = 1
    while n < m["num_constraints"] + ni:
        n *= 2
    m1, m2 = cv.fr([rng.randrange(cv.r) for _ in range(n)]), cv.fr([rng.randrange(cv.r) for _ in range(n)])
    rs = cv.fr([11, 13]), cv.fr([17, 19])

    def locals_of(pk):
        return (pk.rep3_local(0, pub, sh0, m1, m2, *rs), pk.shamir_local(pub, wit, cv.fr([5]), cv.fr([9])))

    full = make_key(emu_ctx, cv, z, m)
    ref_locals = locals_of(full)
    W = full.table_info()[0]
    full.free()
    for k in (2, W):
        pk = key_rows(rows_shim, emu_ctx, cv, z, m, k)
        rows = (W + k - 1) // k
        assert pk.table_info()[0] == rows
        for p in g["oracle_proofs"]:
            r_, s_ = ih(p["r"]), ih(p["s"])
            A, Bp, Cp = pk.prove_plain(pub, wit, cv.fr([r_]), cv.fr([s_]))
            assert (cv.pt1(A), cv.pt2(Bp), cv.pt1(Cp)) == OG.prove_plain(z, m, w, r_, s_), (rows, r_, s_)
        got = locals_of(pk)
        for a, b in zip(got, ref_locals):
            assert all(np.array_equal(x, y) for x, y in zip(a, b)), rows
        pk.free()


def test_groth16_shared_sort_views_compact_emu(emu_ctx, rows_shim):
    """A key with infinity bases in B (the shared witness sort read through filtered views) at k = 2 and one row."""
    cv = Conv("bn254")
    z, m, w, _ = golden_groth16("poseidon")
    nw, ni = m["num_witness_variables"], m["num_instance_variables"]
    assert sum(1 for P in z["b_g1_query"][ni:] if P is None) > 0 and all(P is not None for P in z["l_query"])
    exp = OG.prove_plain(z, m, w, 3, 4)
    pub, wit = cv.fr(w[:ni]), cv.fr(w[ni:])
    full = make_key(emu_ctx, cv, z, m)
    W = full.table_info()[0]
    full.free()
    for k in (2, W):
        pk = key_rows(rows_shim, emu_ctx, cv, z, m, k)
        assert pk.table_info()[0] == (W + k - 1) // k
        A, Bp, Cp = pk.prove_plain(pub, wit, cv.fr([3]), cv.fr([4]))
        assert (cv.pt1(A), cv.pt2(Bp), cv.pt1(Cp)) == exp, k
        pk.free()
    assert nw > 0


def test_table_budget_semantics_emu(emu_ctx, rows_shim, budget_reset):
    """Reported bytes stay within the budget; a budget at least the full tables' gives T = W; a budget below one row
    fails with CS_ERR_LIMIT, stating the bytes, and leaks nothing."""
    budget_reset(emu_ctx)
    cv = Conv("bn254")
    n = 1000
    pts = dlog_bases(emu_ctx, cv, 0, [i + 1 for i in range(n)])
    b = emu_ctx.bases_upload(cv.id, 0, pts)
    info = b.info()
    b.free()
    W, full = info["windows"], info["device_bytes"]
    assert info["table_rows"] == W and info["window_bits"] == auto_window(n, 254)
    for budget in (full, full + 12345, 3 * full):
        emu_ctx.set_table_budget(budget)
        b = emu_ctx.bases_upload(cv.id, 0, pts)
        assert b.info()["table_rows"] == W and b.info()["device_bytes"] <= budget
        b.free()
    for budget in (full // 2, full // 3, full // 5):
        emu_ctx.set_table_budget(budget)
        b = emu_ctx.bases_upload(cv.id, 0, pts)
        assert b.info()["table_rows"] < W and b.info()["device_bytes"] <= budget
        b.free()
    # below one row: CS_ERR_LIMIT with the bytes, and nothing left allocated.  The key's matrices are padded to 2 x 20000
    # entries (about 1.4 MB on the "device", which the emulation takes from the process heap) so that buffers a failed
    # creation kept would show in the heap reading.
    z, m, _, _ = golden_groth16("multiplier2")
    m = dict(m, a=[m["a"][0] + [(0, 0)] * 20000] + m["a"][1:], b=[m["b"][0] + [(0, 0)] * 20000] + m["b"][1:])
    heap = []
    for _ in range(6):
        emu_ctx.set_table_budget(n * 64 // 2)  # less than one row of n 64-byte points
        with pytest.raises(B.CsError, match="bytes") as e:
            emu_ctx.bases_upload(cv.id, 0, pts)
        assert "error %d" % ERR_LIMIT in str(e.value)
        emu_ctx.set_table_budget(1000)
        with pytest.raises(B.CsError, match="error %d" % ERR_LIMIT):
            make_key(emu_ctx, cv, z, m)
        heap.append(rows_shim.heap_bytes_in_use())
    assert heap[-1] - heap[1] < 256 << 10, ("a failed creation leaked device memory", heap)
    emu_ctx.set_table_budget(0)
    z, m, _, _ = golden_groth16("multiplier2")
    pk = make_key(emu_ctx, cv, z, m)
    rows, tb = pk.table_info()
    assert rows == windows(cv, auto_window(m["num_witness_variables"], 254)) and tb > 0
    pk.free()


# ------------------------------------------------------------------------------------------------ GPU
def alloc_size(nbytes):
    """DevBuf::alloc_size (csrc/cs_common.cuh): what the library allocates for nbytes"""
    return nbytes + (nbytes >> 3) + 256


def bases_budget(cv, group, n, rows):
    """the budget at which cs_bases_upload keeps `rows` rows of n points: the smallest k with ceil(W / k) = rows"""
    pb = 8 * cv.nq * (2 if group == 0 else 4)
    return alloc_size(rows * n * pb) + alloc_size((n + 31) // 32 * 4)


@pytest.mark.gpu
@pytest.mark.parametrize("curve", ["bn254", "bls12_381"])
@pytest.mark.parametrize("group", [0, 1])
@pytest.mark.parametrize("lg", [16, 20])
def test_compact_msm_equals_full_gpu(gpu_ctx, budget_reset, curve, group, lg):
    """k in {2, 4, 16} (8, 4 and 1 table rows) bit-identical to the full table; at 2^20 with k = 4 also equal to the
    known discrete-log result."""
    budget_reset(gpu_ctx)
    cv = Conv(curve)
    rng = np.random.default_rng(lg * 10 + group)
    n = 1 << lg
    if lg == 20 and group == 0:
        pyr = random.Random(lg)
        ks = base_dlogs(cv, n, pyr)
        pts = dlog_bases(gpu_ctx, cv, group, ks)
    else:
        ks = None
        gen = B.ints_to_limbs([rng.integers(1, 1 << 62) for _ in range(n)], 4)
        cd = CURVES[curve]
        base = (cv.g1 if group == 0 else cv.g2)([cd.g1 if group == 0 else cd.g2])[0]
        pts = gpu_ctx.fixed_base_mul(cv.id, group, base, gen, montgomery=False)
    sc = rng.integers(0, 1 << 63, size=(n, 4), dtype=np.uint64)
    sc[:, 3] &= np.uint64((1 << 60) - 1)  # < r on both curves
    sc[::97] = 0
    full = gpu_ctx.bases_upload(cv.id, group, pts)
    W = full.info()["windows"]
    assert W == 16 and full.info()["table_rows"] == 16
    ref = [gpu_ctx.msm(full, sc)[0], gpu_ctx.msm(full, sc, montgomery=False)[0]]
    full.free()
    for k in (2, 4, 16):
        rows = (W + k - 1) // k
        gpu_ctx.set_table_budget(bases_budget(cv, group, n, rows))
        b = gpu_ctx.bases_upload(cv.id, group, pts)
        assert b.info()["table_rows"] == rows
        got = [gpu_ctx.msm(b, sc)[0], gpu_ctx.msm(b, sc, montgomery=False)[0]]
        b.free()
        assert all(np.array_equal(x, y) for x, y in zip(got, ref)), ("k", k)
        if ks is not None and k == 4:
            ss = B.limbs_to_ints(sc)
            assert cv.pt1(got[1]) == expected(cv, group, ks, ss)
    gpu_ctx.set_table_budget(0)


def _syn_key(ctx, syn):
    return B.Groth16Key(ctx, syn.cid, syn.matrices, syn.points)


@pytest.mark.gpu
@pytest.mark.parametrize("curve", ["bn254", "bls12_381"])
def test_trapdoor_compact_keys_gpu(gpu_ctx, budget_reset, curve):
    """The known-trapdoor reference at 2^20 through keys the budget forces to k = 2 and k = 4."""
    from test_groth16_trapdoor import device_proof, trapdoor_proof
    from workloads.synth_groth16 import SynthGroth16
    budget_reset(gpu_ctx)
    syn = SynthGroth16(gpu_ctx, 20, curve=curve, keep_trapdoor=True)
    exp = trapdoor_proof(syn, 31337, 271828)
    for rows in (8, 4):
        pk = forced_key(gpu_ctx, lambda: _syn_key(gpu_ctx, syn), rows)
        gpu_ctx.set_table_budget(0)
        assert pk.table_info()[0] == rows  # k = 2, then k = 4
        assert device_proof(syn, pk, 31337, 271828) == exp, rows
        pk.free()
    syn.points = None


@pytest.mark.gpu
def test_rep3_and_shamir_compact_keys_gpu(gpu_ctx):
    """BN254 at 2^16 with eight table rows (k = 2; at this size the scratch of k = 4 outweighs the rows it saves, so no
    budget picks it): Rep3 (three party threads, one GPU) and Shamir(3, 1) proofs open to
    the trapdoor proof for their (r, s)."""
    from test_groth16_trapdoor import trapdoor_proof
    from workloads.synth_groth16 import SynthGroth16
    syn = SynthGroth16(gpu_ctx, 16, keep_trapdoor=True)
    cv = Conv(syn.curve)
    r, ni = syn.r, syn.ni
    nw = len(syn.witness) - ni
    ctxs = [B.Context(0) for _ in range(3)]
    pks = [forced_key(c, lambda c=c: _syn_key(c, syn), 8) for c in ctxs]
    try:
        assert all(pk.table_info()[0] == 8 for pk in pks)
        lib = ctxs[0].lib
        # Rep3
        nets0 = [B.Net.peer(ctxs[i], i, 3) for i in range(3)]
        nets1 = [B.Net.peer(ctxs[i], i, 3) for i in range(3)]
        for i in range(3):
            nets0[i].connect_local(nets0)
            nets1[i].connect_local(nets1)
        seeds = [bytes([31 * (i + 1) + k for k in range(32)]) for i in range(3)]
        states = [B.Rep3StateC.from_seeds(lib, i, seeds[i], seeds[(i + 2) % 3]) for i in range(3)]
        wsh = OG.share_rep3(syn.witness[ni:], r, random.Random(5))
        shares = [syn.fr([x for ab in wsh[i] for x in ab]).reshape(-1, 8) for i in range(3)]
        out, errs = {}, []

        def rep3(i):
            try:
                A, Bp, Cp, rs = pks[i].rep3_prove(nets0[i], nets1[i], states[i], syn.public_inputs, shares[i], want_rs=True)
                out[i] = ((cv.pt1(A), cv.pt2(Bp), cv.pt1(Cp)), cv.fr_back(rs))
            except Exception as e:  # noqa: BLE001
                errs.append(e)
        _run3(rep3)
        assert not errs, errs
        rs = [out[i][1] for i in range(3)]
        r_tot, s_tot = sum(x[0] for x in rs) % r, sum(x[2] for x in rs) % r
        assert out[0][0] == out[1][0] == out[2][0] == trapdoor_proof(syn, r_tot, s_tot), "Rep3"
        for x in nets0 + nets1 + states:
            x.free()
        # Shamir(3, 1)
        nets0 = [B.Net.peer(ctxs[i], i, 3) for i in range(3)]
        nets1 = [B.Net.peer(ctxs[i], i, 3) for i in range(3)]
        for i in range(3):
            nets0[i].connect_local(nets0)
            nets1[i].connect_local(nets1)
        srng = random.Random(6)
        coef = [srng.randrange(r) for _ in range(nw)]
        wsh = [[(x + c * (i + 1)) % r for x, c in zip(syn.witness[ni:], coef)] for i in range(3)]  # degree 1 at x = 1, 2, 3
        out, errs = {}, []

        def shamir(i):
            try:
                A, Bp, Cp, rs = pks[i].shamir_prove(nets0[i], nets1[i], 3, 1, syn.public_inputs, syn.fr(wsh[i]))
                out[i] = ((cv.pt1(A), cv.pt2(Bp), cv.pt1(Cp)), cv.fr_back(rs))
            except Exception as e:  # noqa: BLE001
                errs.append(e)
        _run3(shamir)
        assert not errs, errs
        assert out[0][0] == out[1][0] == out[2][0], "Shamir parties disagree"
        lag = [3, r - 3, 1]  # Lagrange coefficients at 0 of the points 1, 2, 3
        r_tot = sum(l * out[i][1][0] for i, l in enumerate(lag)) % r
        s_tot = sum(l * out[i][1][1] for i, l in enumerate(lag)) % r
        assert out[0][0] == trapdoor_proof(syn, r_tot, s_tot), "Shamir"
        for x in nets0 + nets1:
            x.free()
    finally:
        for pk in pks:
            pk.free()
        for c in ctxs:
            c.set_table_budget(0)
            c.close()
        syn.points = None


def _run3(fn):
    th = [threading.Thread(target=fn, args=(i,)) for i in range(3)]
    for t in th:
        t.start()
    for t in th:
        t.join(timeout=900)


@pytest.mark.gpu
def test_bn254_2_24_key_without_budget_gpu(gpu_ctx):
    """The capability: a BN254 key of 2^24 constraints, whose full tables (about 108 GB with the allocator's slack) do not
    fit an 80 GB H100, created with no budget set.  Fewer rows than windows are chosen automatically, and the plain
    proof equals oracle/c's prove_plain byte for byte on the same key, witness and (r, s).  About 330 s on an H100 80GB
    HBM3 box with 8 host cores, most of it oracle/c's proof and the key's host-side construction."""
    from oracle.c import run as OC
    mats, pts, pub, wit = random_key(gpu_ctx, 24)
    pk = B.Groth16Key(gpu_ctx, B.CS_BN254, mats, pts)
    try:
        rows, tbytes = pk.table_info()
        assert rows < 16, rows
        r_, s_ = rand_fr_limbs(np.random.default_rng(1), 2)
        got = pk.prove_plain(pub, wit, r_[None, :].copy(), s_[None, :].copy())
    finally:
        pk.free()
    desc, keep = OC.key_desc(mats, pts, curve=B.CS_BN254)
    exp = OC.prove_plain(desc, pub, wit, r_[None, :].copy(), s_[None, :].copy())
    del keep
    for g, e, name in zip(got, exp, "ABC"):
        assert np.array_equal(np.asarray(g).reshape(-1), np.asarray(e).reshape(-1)), name
