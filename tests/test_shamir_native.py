"""Shamir(n, t) inside the library (csrc/cs_shamir.cu): preprocessing of DN07 double sharings, king-based degree
reduction of vectors and points, openings, ShamirCoGroth16::prove and the Rep3 -> Shamir bridge.

Mirrors tests/tests/circom/e2e_tests/shamir.rs:37-91 (all parties return the same proof and it verifies) and adds
byte parity with the oracle's plain proof for r = r(0), s = s(0); the degree reduction is exercised on the
scalar_mul leg of the prover (degree_reduce_point) and on vectors with n = 5, t = 2, where the king, the senders, the
receivers and the zero-share parties are all distinct roles (mpc-core/src/protocols/shamir/network.rs:150-243).
Parties are threads over in-process mailbox nets; CPU runs use the emulation build."""
import ctypes as C
import os
import random
import sys
import threading

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _emu_factory():
    from co_snarks_b200 import binding as B
    sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
    import build_emu
    emu = build_emu.build()
    return lambda: B.Context(0, lib_path=emu)


def _mesh(ctxs, n, count=1):
    from co_snarks_b200 import binding as B
    nets = [[B.Net.peer(ctxs[i], i, n) for i in range(n)] for _ in range(count)]
    for row in nets:
        for net in row:
            net.connect_local(row)
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


def _run(th):
    for t in th:
        t.start()
    for t in th:
        t.join(timeout=600)


def _degree_reduce_vectors(mk, n, t, length):
    """x, y shared with degree t; local products are degree 2t; after degree_reduce_many the shares are degree t again
    and any t + 1 of them reconstruct x * y."""
    from co_snarks_b200 import binding as B
    from helpers import Conv
    cv = Conv("bn254")
    r = cv.r
    rng = random.Random(7)
    ctxs = [mk() for _ in range(n)]
    lib = ctxs[0].lib
    (nets,) = _mesh(ctxs, n)
    xs = [rng.randrange(r) for _ in range(length)]
    ys = [rng.randrange(r) for _ in range(length)]

    def share(vals):
        out = [[] for _ in range(n)]
        for v in vals:
            co = [v] + [rng.randrange(r) for _ in range(t)]
            for i in range(n):
                out[i].append(sum(c * pow(i + 1, k, r) for k, c in enumerate(co)) % r)
        return out
    xsh, ysh = share(xs), share(ys)
    res, errs = {}, []

    def party(i):
        try:
            ctx = ctxs[i]
            h = C.c_void_p()
            ctx._check(lib.cs_shamir_state_create(nets[i].h, cv.id, n, t, 4, C.byref(h)))
            assert lib.cs_shamir_state_pairs(h) >= 4
            dx, dy = ctx.to_device(cv.fr(xsh[i])), ctx.to_device(cv.fr(ysh[i]))
            ctx._check(lib.cs_vec_mul(ctx.h, cv.id, dx, dy, dx, length))       # local_mul_vec: degree 2t
            ctx._check(lib.cs_shamir_degree_reduce_many(ctx.h, h, nets[i].h, dx, length, dy))
            res[i] = cv.fr_back(ctx.d2h(dy, (length, 4)))
            # ShamirState::rand: a degree-t sharing of a value nobody knows
            sh = np.zeros(4, dtype=np.uint64)
            ctx._check(lib.cs_shamir_state_rand(h, nets[i].h, B._ptr(sh)))
            res[("rand", i)] = cv.fr_back(sh)[0]
            lib.cs_shamir_state_free(h)
            ctx.free(dx)
            ctx.free(dy)
        except Exception as e:  # noqa: BLE001
            errs.append(e)
    _run([threading.Thread(target=party, args=(i,)) for i in range(n)])
    assert not errs, errs
    exp = [x * y % r for x, y in zip(xs, ys)]
    # the last t parties hold zero shares of the king's re-sharing, minus their r_t share: still a valid degree-t sharing
    for subset in ([0, 1, 2][:t + 1], list(range(n - t - 1, n)), [0, n - 1] + list(range(1, t))):
        subset = sorted(set(subset))[:t + 1]
        if len(subset) < t + 1:
            continue
        lam = _lagrange_at_zero([i + 1 for i in subset], r)
        got = [sum(l * res[i][k] for l, i in zip(lam, subset)) % r for k in range(length)]
        assert got == exp, subset
    # the random sharing is consistent: every (t + 1)-subset reconstructs the same value
    vals = set()
    for subset in (list(range(t + 1)), list(range(n - t - 1, n))):
        lam = _lagrange_at_zero([i + 1 for i in subset], r)
        vals.add(sum(l * res[("rand", i)] for l, i in zip(lam, subset)) % r)
    assert len(vals) == 1
    for net in nets:
        net.free()
    for c in ctxs:
        c.close()


def _shamir_groth16(mk, name, n=3, t=1, bridge=False, curve="bn254"):
    from helpers import Conv, golden_groth16, ih, make_key
    from kernel_checks import groth16_verifier
    from oracle import groth16 as OG
    groth16_verify = groth16_verifier(curve)
    cv = Conv(curve)
    r = cv.r
    z, m, w, g = golden_groth16(name, curve)
    ni = m["num_instance_variables"]
    pub = cv.fr(w[:ni])
    ctxs = [mk() for _ in range(n)]
    pks = [make_key(c, cv, z, m) for c in ctxs]
    nets0, nets1 = _mesh(ctxs, n, 2)
    rng = random.Random(77)
    if bridge:
        wsh = OG.share_rep3(w[ni:], r, rng)
        inputs = [cv.fr([x for ab in wsh[i] for x in ab]).reshape(-1, 8) for i in range(3)]
    else:
        co = [[v] + [rng.randrange(r) for _ in range(t)] for v in w[ni:]]
        inputs = [cv.fr([sum(c * pow(i + 1, k, r) for k, c in enumerate(cs)) % r for cs in co]) for i in range(n)]
    out, errs = {}, []

    def party(i):
        try:
            if bridge:
                out[i] = pks[i].prove_with_shamir_bridge(nets0[i], nets1[i], pub, inputs[i])
            else:
                out[i] = pks[i].shamir_prove(nets0[i], nets1[i], n, t, pub, inputs[i])
        except Exception as e:  # noqa: BLE001
            errs.append(e)
    _run([threading.Thread(target=party, args=(i,)) for i in range(n)])
    assert not errs, errs
    proofs = [(cv.pt1(out[i][0]), cv.pt2(out[i][1]), cv.pt1(out[i][2])) for i in range(n)]
    assert all(p == proofs[0] for p in proofs), "parties disagree on the proof"
    assert groth16_verify(OG.vk_from_zkey(z), [ih(x) for x in g["public"]], proofs[0])
    # r, s are degree-t sharings: any t + 1 parties' shares give r(0), s(0); the proof is the plain one for them
    rs = [cv.fr_back(out[i][3]) for i in range(n)]
    lam = _lagrange_at_zero(list(range(1, t + 2)), r)
    r0 = sum(l * rs[i][0] for i, l in enumerate(lam)) % r
    s0 = sum(l * rs[i][1] for i, l in enumerate(lam)) % r
    lam2 = _lagrange_at_zero(list(range(n - t, n + 1)), r)
    assert r0 == sum(l * rs[n - t - 1 + k][0] for k, l in enumerate(lam2)) % r
    assert proofs[0] == OG.prove_plain(z, m, w, r0, s0), "opened Shamir proof != plain proof for r(0), s(0)"
    sent = [x.bytes_sent for x in nets0 + nets1]
    assert all(0 < b < 4096 for b in sent)  # pairs, points and nothing vector-sized
    for pk in pks:
        pk.free()
    for net in nets0 + nets1:
        net.free()
    for c in ctxs:
        c.close()


def test_shamir_degree_reduce_many_n5_t2_emu():
    _degree_reduce_vectors(_emu_factory(), 5, 2, 37)


def test_shamir_degree_reduce_many_n3_t1_emu():
    _degree_reduce_vectors(_emu_factory(), 3, 1, 20)


def test_shamir_dealing_larger_than_the_credit_window_emu():
    # 20000 pairs at t = 1 are 10000 dealings of 64 B per party pair = 640 KB > 8 x 64 KB of mailbox credit: every party
    # deals to every other at the same time (cs_net_sendrecv), then degree-reduces a vector of 640 KB through the king
    _degree_reduce_vectors(_emu_factory(), 3, 1, 20000)


def test_shamir_co_groth16_native_emu():
    _shamir_groth16(_emu_factory(), "multiplier2")


def test_shamir_co_groth16_native_n5_t2_emu():
    _shamir_groth16(_emu_factory(), "multiplier2", n=5, t=2)


def test_groth16_prove_with_shamir_bridge_emu():
    _shamir_groth16(_emu_factory(), "multiplier2", bridge=True)


@pytest.mark.parametrize("name", ["multiplier2", "poseidon"])
def test_shamir_co_groth16_native_bls12_381_emu(name):
    _shamir_groth16(_emu_factory(), name, curve="bls12_381")


@pytest.mark.parametrize("name", ["multiplier2", "poseidon"])
def test_groth16_prove_with_shamir_bridge_bls12_381_emu(name):
    _shamir_groth16(_emu_factory(), name, bridge=True, curve="bls12_381")


def test_shamir_state_rejects_large_threshold_emu():
    from co_snarks_b200 import binding as B
    mk = _emu_factory()
    ctxs = [mk() for _ in range(3)]
    (nets,) = _mesh(ctxs, 3)
    h = C.c_void_p()
    assert ctxs[0].lib.cs_shamir_state_create(nets[0].h, B.CS_BN254, 3, 2, 0, C.byref(h)) != 0
    assert b"Threshold too large for number of parties" in ctxs[0].lib.cs_last_error()


@pytest.mark.gpu
def test_shamir_degree_reduce_many_gpu():
    from co_snarks_b200 import binding as B
    _degree_reduce_vectors(lambda: B.Context(0), 5, 2, 70000)  # > one 64 KB mailbox slot, > the credit window


@pytest.mark.gpu
def test_shamir_co_groth16_native_gpu():
    from co_snarks_b200 import binding as B
    _shamir_groth16(lambda: B.Context(0), "poseidon")


@pytest.mark.gpu
def test_groth16_prove_with_shamir_bridge_gpu():
    from co_snarks_b200 import binding as B
    _shamir_groth16(lambda: B.Context(0), "poseidon", bridge=True)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["multiplier2", "poseidon"])
def test_shamir_co_groth16_native_bls12_381_gpu(name):
    from co_snarks_b200 import binding as B
    _shamir_groth16(lambda: B.Context(0), name, curve="bls12_381")


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["multiplier2", "poseidon"])
def test_groth16_prove_with_shamir_bridge_bls12_381_gpu(name):
    from co_snarks_b200 import binding as B
    _shamir_groth16(lambda: B.Context(0), name, bridge=True, curve="bls12_381")
