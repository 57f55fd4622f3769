"""ShamirCoPlonk::prove inside the library (cs_plonk_shamir_prove, co-plonk/src/lib.rs:237-260) and the device double
sharings it consumes (cs_shamir_double_sharings).

Parties are threads over in-process mailbox nets, each with its own context, key and session.  Checks:
 * device pairs: every (t + 1)-subset of r_t shares and every (2t + 1)-subset of r_2t shares reconstruct the same
   value, the two agree, and no value repeats across two calls (a reused dealing seed would repeat them);
 * known answer: with degree-t sharings of b = [0..11) the opened proof is the reference's round 1-5 answer;
 * drawn blinders: the opened proof is the plain prover's for the blinders the parties' shares reconstruct to;
 * accounting: pairs per proof and bytes per party match the documented formula; bad arguments are refused.
CPU runs use the emulation build."""
import ctypes as C
import itertools
import os
import random
import sys
import threading

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ERR_ARG, ERR_LIMIT = -1, -3  # CS_ERR_ARG, CS_ERR_LIMIT (include/cosnarks_gpu.h)


def _emu_factory():
    from co_snarks_b200 import binding as B
    sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
    import build_emu
    emu = build_emu.build()
    return lambda: B.Context(0, lib_path=emu)


def _gpu_factory():
    from co_snarks_b200 import binding as B
    return lambda: B.Context(0)


def _nets(ctxs, n):
    from co_snarks_b200 import binding as B
    nets = [B.Net.peer(ctxs[i], i, n) for i in range(n)]
    for net in nets:
        net.connect_local(nets)
    return nets


def _lagrange_at_zero(points, r):
    out = []
    for i in points:
        num, den = 1, 1
        for j in points:
            if j != i:
                num = num * j % r
                den = den * (j - i) % r
        out.append(num * pow(den, -1, r) % r)
    return out


def _reconstruct(shares, subset, r):
    """shares[p] = party p's value; subset: party ids (evaluation points p + 1)"""
    lam = _lagrange_at_zero([p + 1 for p in subset], r)
    return sum(l * shares[p] for l, p in zip(lam, subset)) % r


def _share(vals, n, t, r, rng):
    out = [[] for _ in range(n)]
    for v in vals:
        co = [v] + [rng.randrange(r) for _ in range(t)]
        for i in range(n):
            out[i].append(sum(c * pow(i + 1, k, r) for k, c in enumerate(co)) % r)
    return out


def _threads(fn, n):
    errs = []

    def run(p):
        try:
            fn(p)
        except Exception as e:  # noqa: BLE001
            errs.append(e)
    th = [threading.Thread(target=run, args=(p,)) for p in range(n)]
    for t in th:
        t.start()
    for t in th:
        t.join(timeout=1800)
    assert not errs, errs


def _subsets(n, k, limit=12):
    return list(itertools.combinations(range(n), k))[:limit]


# ---- 1. device double sharings ------------------------------------------------------------------------------------

def _device_pairs(mk, n, t, curve, counts):
    from helpers import Conv
    cv = Conv(curve)
    r = cv.r
    ctxs = [mk() for _ in range(n)]
    lib = ctxs[0].lib
    nets = _nets(ctxs, n)
    res = {}

    def party(p):
        ctx = ctxs[p]
        h = C.c_void_p()
        ctx._check(lib.cs_shamir_state_create(nets[p].h, cv.id, n, t, 0, C.byref(h)))
        out = []
        for cnt in counts:
            drt, dr2t = ctx.to_device(np.zeros((cnt, 4), dtype=np.uint64)), ctx.to_device(np.zeros((cnt, 4), dtype=np.uint64))
            ctx._check(lib.cs_shamir_double_sharings(ctx.h, h, nets[p].h, cnt, drt, dr2t))
            out.append((cv.fr_back(ctx.d2h(drt, (cnt, 4))), cv.fr_back(ctx.d2h(dr2t, (cnt, 4)))))
            ctx.free(drt)
            ctx.free(dr2t)
        lib.cs_shamir_state_free(h)
        res[p] = out
    _threads(party, n)
    seen = set()
    for c, cnt in enumerate(counts):
        for i in range(cnt):
            rt = {p: res[p][c][0][i] for p in range(n)}
            r2t = {p: res[p][c][1][i] for p in range(n)}
            vt = {_reconstruct(rt, s, r) for s in _subsets(n, t + 1)}
            v2t = {_reconstruct(r2t, s, r) for s in _subsets(n, 2 * t + 1)}
            assert len(vt) == 1, ("r_t is not a degree-t sharing", c, i)
            assert len(v2t) == 1, ("r_2t is not a degree-2t sharing", c, i)
            assert vt == v2t, ("r_t and r_2t share different values", c, i)
            seen.add(vt.pop())
    assert len(seen) == sum(counts), "a double sharing repeats"
    # r_2t is not a degree-t sharing (it would be if the g dealing had degree t)
    rt0 = {p: res[p][0][1][0] for p in range(n)}
    assert len({_reconstruct(rt0, s, r) for s in _subsets(n, t + 1)}) > 1
    for net in nets:
        net.free()
    for c in ctxs:
        c.close()


@pytest.mark.parametrize("curve", ["bn254", "bls12_381"])
@pytest.mark.parametrize("n,t", [(4, 1), (5, 2)])
def test_device_double_sharings_emu(n, t, curve):
    _device_pairs(_emu_factory(), n, t, curve, [37, 20])


@pytest.mark.gpu
@pytest.mark.parametrize("curve", ["bn254", "bls12_381"])
@pytest.mark.parametrize("n,t", [(4, 1), (5, 2)])
def test_device_double_sharings_gpu(n, t, curve):
    _device_pairs(_gpu_factory(), n, t, curve, [20001, 3])  # > the mailbox credit window per dealing


# ---- 2-5. proofs ----------------------------------------------------------------------------------------------------

def _pair_formula(dom, drawn):
    return 58 * dom + 2 + (11 if drawn else 0)


def _bytes_bound(dom, n, t):
    """Upper bound on what one party sends in a proof: dealings of the two device pair rounds, the 55 dom reductions
    (the king sends the most), the three openings of n-sized degree-2t vectors, and 256 KB for the host pool the
    blinders come from, the points and the scalars."""
    deal = lambda cnt: 64 * (n - 1) * -(-cnt // (t + 1))
    return (deal(10 * dom + 2) + deal(48 * dom) + 32 * max(n - t - 1, 1) * 55 * dom + 64 * t * (3 * dom + 1)
            + 256 * 1024)


def _prove(mk, n, t, curve, z=None, w=None, key=None, fixed_blinders=True, seed=5):
    """-> (proofs per party as oracle dicts, blinder shares per party, sessions' pair counts, bytes sent, pk, ctxs...)"""
    from co_snarks_b200 import binding as B
    from helpers import Conv, make_plonk_key, plonk_proof_from_device
    cv = Conv(curve)
    r = cv.r
    rng = random.Random(seed)
    npub = key["n_public"] if key else z["n_public"]
    pub = cv.fr(w[:npub + 1])
    wsh = [cv.fr(s) for s in _share(w[npub + 1:], n, t, r, rng)]
    bsh = [cv.fr(s) for s in _share(list(range(11)), n, t, r, rng)] if fixed_blinders else [None] * n
    ctxs = [mk() for _ in range(n)]
    pks = [B.PlonkKey(c, cv.id, key) if key else make_plonk_key(c, cv, z) for c in ctxs]
    sess = [B.PlonkShamirSession(ctxs[p], pks[p], n, t, p) for p in range(n)]
    nets = _nets(ctxs, n)
    res = {}

    def party(p):
        res[p] = sess[p].prove(nets[p], pub, wsh[p], bsh[p])
    _threads(party, n)
    proofs = [plonk_proof_from_device(cv, *res[p][:2]) for p in range(n)]
    bl = [cv.fr_back(res[p][2]) for p in range(n)]
    out = dict(proofs=proofs, blinders=bl, pairs=[s.pairs() for s in sess], sent=[x.bytes_sent for x in nets],
               pub=pub, ctx0=ctxs[0], pk0=pks[0], cv=cv)
    if fixed_blinders:
        assert all(np.array_equal(res[p][2], bsh[p]) for p in range(n))

    def close():
        for s in sess:
            s.free()
        for pk in pks:
            pk.free()
        for x in nets:
            x.free()
        for c in ctxs:
            c.close()
    out["close"] = close
    return out


def _verify(curve, z, g, proof):
    from helpers import ih, plonk_vk_from_zkey
    from oracle import plonk as OP
    from oracle.fields import CURVES
    if curve == "bn254":
        from oracle.pairing_bn254 import pairing_product_is_one
    else:
        from oracle.pairing_bls12_381 import pairing_product_is_one
    return OP.verify(CURVES[curve], plonk_vk_from_zkey(z, g["vk_power"]), proof, [ih(x) for x in g["public"]],
                     pairing_product_is_one)


def _kat(mk, name, curve, n=3, t=1):
    from helpers import golden_plonk
    from oracle.formats import plonk_proof_to_json
    z, w, g = golden_plonk(name, curve)
    o = _prove(mk, n, t, curve, z=z, w=w, fixed_blinders=True)
    try:
        p = o["proofs"]
        assert all(x == p[0] for x in p), "parties disagree on the proof"
        assert plonk_proof_to_json(p[0], g["oracle_proof_json"]["curve"]) == g["oracle_proof_json"]
        assert _verify(curve, z, g, p[0])
        dom = z["domain_size"]
        assert o["pairs"] == [_pair_formula(dom, False)] * n
        assert all(0 < s <= _bytes_bound(dom, n, t) for s in o["sent"]), o["sent"]
    finally:
        o["close"]()


def _drawn(mk, name, curve, n, t):
    """Blinders drawn by the parties: reconstructed from two (t + 1)-subsets, the opened proof is the plain prover's
    for them, byte for byte, and verifies."""
    from helpers import golden_plonk
    z, w, g = golden_plonk(name, curve)
    o = _prove(mk, n, t, curve, z=z, w=w, fixed_blinders=False)
    try:
        cv, r = o["cv"], o["cv"].r
        p = o["proofs"]
        assert all(x == p[0] for x in p), "parties disagree on the proof"
        sh = o["blinders"]
        b = [_reconstruct({q: sh[q][i] for q in range(n)}, list(range(t + 1)), r) for i in range(11)]
        b2 = [_reconstruct({q: sh[q][i] for q in range(n)}, list(range(n - t - 1, n)), r) for i in range(11)]
        assert b == b2, "blinder shares are not a degree-t sharing"
        assert len(set(b)) == 11
        npub = z["n_public"]
        pts, evs = o["pk0"].prove_plain(o["pub"], cv.fr(w[npub + 1:]), cv.fr(b))
        from helpers import plonk_proof_from_device
        assert p[0] == plonk_proof_from_device(cv, pts, evs), "opened Shamir proof != plain proof for the same blinders"
        assert _verify(curve, z, g, p[0])
        dom = z["domain_size"]
        assert o["pairs"] == [_pair_formula(dom, True)] * n
        assert all(0 < s <= _bytes_bound(dom, n, t) for s in o["sent"]), o["sent"]
        assert o["sent"][0] >= 32 * (n - t - 1) * 55 * dom  # the king re-shares every reduced product
    finally:
        o["close"]()


def test_plonk_shamir_kat_bn254_multiplier2_emu():
    _kat(_emu_factory(), "multiplier2", "bn254")


def test_plonk_shamir_kat_bls12_381_multiplier2_emu():
    _kat(_emu_factory(), "multiplier2", "bls12_381")


def test_plonk_shamir_drawn_blinders_n5_t2_emu():
    _drawn(_emu_factory(), "multiplier2", "bn254", 5, 2)


@pytest.mark.gpu
def test_plonk_shamir_kat_bn254_poseidon_gpu():
    _kat(_gpu_factory(), "poseidon", "bn254")


@pytest.mark.gpu
def test_plonk_shamir_kat_bls12_381_multiplier2_gpu():
    _kat(_gpu_factory(), "multiplier2", "bls12_381")


@pytest.mark.gpu
def test_plonk_shamir_drawn_blinders_n5_t2_gpu():
    _drawn(_gpu_factory(), "poseidon", "bn254", 5, 2)


def _production(mk, lg):
    """A synthetic 2^lg key on BN254, n = 3, t = 1, drawn blinders: the opened proof equals the plain prover's for the
    reconstructed blinders and passes the pairing check."""
    from helpers import plonk_proof_from_device
    from oracle import plonk as OP
    from oracle.fields import BN254
    from oracle.pairing_bn254 import pairing_product_is_one
    from workloads.synth_plonk import SynthPlonk
    n, t = 3, 1
    ctx = mk()
    syn = SynthPlonk(ctx, lg)
    key, vk, w = syn.key, syn.vk_ints(), list(syn.full_witness)  # witness: leading one, public, private
    ctx.close()
    o = _prove(mk, n, t, "bn254", w=w, key=key, fixed_blinders=False)
    try:
        cv, r = o["cv"], o["cv"].r
        p = o["proofs"]
        assert all(x == p[0] for x in p), "parties disagree on the proof"
        sh = o["blinders"]
        b = [_reconstruct({q: sh[q][i] for q in range(n)}, [0, 1], r) for i in range(11)]
        assert b == [_reconstruct({q: sh[q][i] for q in range(n)}, [1, 2], r) for i in range(11)]
        npub = syn.n_public
        pts, evs = o["pk0"].prove_plain(o["pub"], cv.fr(w[npub + 1:]), cv.fr(b))
        assert p[0] == plonk_proof_from_device(cv, pts, evs), "opened Shamir proof != plain proof"
        assert OP.verify(BN254, vk, p[0], w[1:npub + 1], pairing_product_is_one)
        assert o["pairs"] == [_pair_formula(syn.n, True)] * n
        assert all(0 < s <= _bytes_bound(syn.n, n, t) for s in o["sent"]), o["sent"]
    finally:
        o["close"]()


def test_plonk_shamir_synthetic_2p8_emu():
    _production(_emu_factory(), 8)


@pytest.mark.gpu
def test_plonk_shamir_production_shape_2p18_gpu():
    _production(_gpu_factory(), 18)


# ---- repeated calls hold no memory beyond the reused workspace ---------------------------------------------------------

def _emu_live_bytes():
    """bytes the process's heap holds (glibc mallinfo2 over all arenas, mmapped chunks included): the emulation build
    allocates "device" memory with malloc"""
    class MallInfo2(C.Structure):
        _fields_ = [(f, C.c_size_t) for f in ("arena", "ordblks", "smblks", "hblks", "hblkhd", "usmblks", "fsmblks",
                                               "uordblks", "fordblks", "keepcost")]
    libc = C.CDLL(None)
    libc.mallinfo2.restype = MallInfo2
    m = libc.mallinfo2()
    return m.uordblks + m.hblkhd


def _gpu_used_bytes():
    import torch
    free, total = torch.cuda.mem_get_info(0)
    return total - free


def _double_sharings_flat(mk, used, count, calls, slack):
    """cs_shamir_double_sharings called again and again by n = 3, t = 1 parties: memory after the first call equals
    memory after the last (a call that leaked its staging would grow it by ~12 count / 2 elements per party)."""
    n, t = 3, 1
    from helpers import Conv
    cv = Conv("bn254")
    ctxs = [mk() for _ in range(n)]
    lib = ctxs[0].lib
    nets = _nets(ctxs, n)
    hs = []
    for p in range(n):
        h = C.c_void_p()
        ctxs[p]._check(lib.cs_shamir_state_create(nets[p].h, cv.id, n, t, 0, C.byref(h)))
        hs.append(h)
    bufs = [(c.to_device(np.zeros((count, 4), dtype=np.uint64)), c.to_device(np.zeros((count, 4), dtype=np.uint64))) for c in ctxs]

    def once(p):
        ctxs[p]._check(lib.cs_shamir_double_sharings(ctxs[p].h, hs[p], nets[p].h, count, bufs[p][0], bufs[p][1]))
    _threads(once, n)
    first = used()
    for _ in range(calls - 1):
        _threads(once, n)
    grown = used() - first
    for p in range(n):
        lib.cs_shamir_state_free(hs[p])
        ctxs[p].free(bufs[p][0])
        ctxs[p].free(bufs[p][1])
    for x in nets:
        x.free()
    for c in ctxs:
        c.close()
    assert grown < slack, "memory grew by %d bytes over %d calls" % (grown, calls - 1)


def _proofs_flat(mk, used, lg, proofs, slack):
    """Repeated proofs on the same sessions: memory after the first proof equals memory after the last."""
    from co_snarks_b200 import binding as B
    from helpers import Conv
    from workloads.synth_plonk import SynthPlonk
    n, t = 3, 1
    cv = Conv("bn254")
    ctx = mk()
    syn = SynthPlonk(ctx, lg)
    key, w = syn.key, list(syn.full_witness)
    ctx.close()
    npub = key["n_public"]
    pub = cv.fr(w[:npub + 1])
    wsh = [cv.fr(x) for x in _share(w[npub + 1:], n, t, cv.r, random.Random(3))]
    ctxs = [mk() for _ in range(n)]
    pks = [B.PlonkKey(c, cv.id, key) for c in ctxs]
    sess = [B.PlonkShamirSession(ctxs[p], pks[p], n, t, p) for p in range(n)]
    nets = _nets(ctxs, n)
    res = {}

    def prove(p):
        res[p] = sess[p].prove(nets[p], pub, wsh[p])
    _threads(prove, n)
    first, held = used(), [x.device_bytes() for x in sess]
    for _ in range(proofs - 1):
        _threads(prove, n)
    grown = used() - first
    assert [x.device_bytes() for x in sess] == held and all(b > 0 for b in held)
    assert held[0] > held[1]  # the king stages the 2t received vectors and the Lagrange sum of every reduction
    for x in sess + pks + nets:
        x.free()
    for c in ctxs:
        c.close()
    assert grown < slack, "memory grew by %d bytes over %d proofs" % (grown, proofs - 1)


def test_double_sharings_memory_flat_emu():
    _double_sharings_flat(_emu_factory(), _emu_live_bytes, 200000, 5, 4 << 20)


def test_plonk_shamir_memory_flat_over_proofs_emu():
    _proofs_flat(_emu_factory(), _emu_live_bytes, 8, 4, 1 << 20)


@pytest.mark.gpu
def test_double_sharings_memory_flat_gpu():
    _double_sharings_flat(_gpu_factory(), _gpu_used_bytes, (1 << 21) + 5, 4, 64 << 20)


@pytest.mark.gpu
def test_plonk_shamir_memory_flat_over_proofs_gpu():
    _proofs_flat(_gpu_factory(), _gpu_used_bytes, 16, 3, 64 << 20)


# ---- 5. argument checks ---------------------------------------------------------------------------------------------

def _rejections(mk):
    from co_snarks_b200 import binding as B
    from helpers import Conv, golden_plonk, make_plonk_key
    cv = Conv("bn254")
    z, w, g = golden_plonk("multiplier2")
    ctx = mk()
    lib = ctx.lib
    pk = make_plonk_key(ctx, cv, z)
    h = C.c_void_p()
    assert lib.cs_plonk_shamir_create(ctx.h, pk.h, 3, 0, 0, C.byref(h)) == ERR_ARG        # t = 0
    assert lib.cs_plonk_shamir_create(ctx.h, pk.h, 4, 2, 0, C.byref(h)) == ERR_ARG        # 2t + 1 > n
    assert lib.cs_plonk_shamir_create(ctx.h, pk.h, 9, 1, 0, C.byref(h)) == ERR_LIMIT      # n > 8
    assert lib.cs_plonk_shamir_create(ctx.h, pk.h, 3, 1, 3, C.byref(h)) == ERR_ARG        # party out of range
    npub = z["n_public"]
    pub, wit = cv.fr(w[:npub + 1]), cv.fr(w[npub + 1:])
    pts, evs = np.zeros((9, 8), dtype=np.uint64), np.zeros((6, 4), dtype=np.uint64)
    nets4 = [B.Net.peer(ctx, i, 4) for i in range(4)]
    nets3 = [B.Net.peer(ctx, i, 3) for i in range(3)]
    assert lib.cs_plonk_shamir_prove(None, nets3[0].h, B._ptr(pub), pub.shape[0], B._ptr(wit), wit.shape[0], None,
                                     B._ptr(pts), B._ptr(evs), None) == ERR_ARG           # NULL session
    s = B.PlonkShamirSession(ctx, pk, 3, 1, 0)
    assert lib.cs_plonk_shamir_prove(s.h, nets4[0].h, B._ptr(pub), pub.shape[0], B._ptr(wit), wit.shape[0], None,
                                     B._ptr(pts), B._ptr(evs), None) == ERR_ARG           # net of 4 parties
    assert lib.cs_plonk_shamir_prove(s.h, nets3[1].h, B._ptr(pub), pub.shape[0], B._ptr(wit), wit.shape[0], None,
                                     B._ptr(pts), B._ptr(evs), None) == ERR_ARG           # net of party 1
    assert s.pairs() == 0
    s.free()
    for x in nets3 + nets4:
        x.free()
    pk.free()
    ctx.close()


def test_plonk_shamir_rejects_bad_arguments_emu():
    _rejections(_emu_factory())


@pytest.mark.gpu
def test_plonk_shamir_rejects_bad_arguments_gpu():
    _rejections(_gpu_factory())
