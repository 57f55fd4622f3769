"""Plonk proofs checked exactly against what the known trapdoor tau implies, on BN254 and BLS12-381, plain, Rep3 and
Shamir, at the sizes production runs.

workloads/synth_plonk.py builds the key from a known tau and keeps the values the key interpolates: the selectors and
sigmas on H, the wire values and the domain.  For x not in H the reference evaluates any polynomial given by its values
on H with the barycentric form L_i(x) = w^i (x^n - 1) / (n (x - w^i)), one batch inversion per point, in O(n) python
integer work and without an NTT or an MSM.  With the blinders b[0..11) and the conventions of oracle/plonk.py
(a(X) = sum A_i L_i(X) + (b0 X + b1) Z_H(X), likewise b, c, and z with b6 X^2 + b7 X + b8), it checks, in transcript
order so that every point is checked before a challenge derived from it is used:
  * [A], [B], [C], [Z] = p(tau) G1;
  * [T1] + tau^n [T2] + tau^2n [T3] = t(tau) G1, t(tau) = (the quotient identity at tau) / Z_H(tau);
  * the six evaluations a, b, c, s1, s2 at xi and z at xi w;
  * (tau - xi w) [W_xiw] = (z(tau) - z(xi w)) G1;
  * (tau - xi) [W_xi] = S G1 - Z_H(xi) ([T1] + xi^n [T2] + xi^2n [T3]), S the round-5 polynomial of oracle/plonk.py at
    tau without its T part (it vanishes at xi for a correct proof, so nothing is lost to the division);
  * the verification key: q_k(tau) G1 and sigma_k(tau) G1.
The challenges are recomputed with oracle.plonk.Transcript from the proof's own points.  The reference does not pin how
t is split into T1, T2, T3 (the b9 / b10 blinders cancel in the T sum); exact equality with oracle/c (BN254) and with
oracle/plonk.py (small sizes, both curves) pins that, and a negative control below shows the gap.  The rest of the key
is checked independently of the device: coefficients and 4n-point evaluations against oracle/c's NTT, p_tau at its
ends and at 64 random indices against oracle.ec.

`gates="mixed"` draws full-width selectors per row, with linear rows and rows without q_L / q_R, so a kernel that used
the wrong selector for a wire or lost a carry of a full-width selector fails here; the fixed gates leave q_R zero.

GPU keys live in class-scoped fixtures and are freed when their class is done.  Wall time and peak device memory per
case, measured on an 80 GB H100 (peak = total - free sampled every 20 ms, so it includes the test's CUDA contexts and
any other work on the card):
  BN254 2^20 mixed   key build 81 s, reference at tau 13 s, key vs oracle/c 40 s, proof 0.6 s (6.6 GB),
                     reference checks 28 s, oracle/c plonk_prove 38 s
  BN254 2^22 fixed   key build 95 s, reference at tau 43 s, key vs oracle/c 126 s, proof 2.3 s (22.4 GB),
                     reference checks 94 s
  BN254 2^21 Rep3    key build 53 s, reference at tau 25 s, three-party proof 28 s (72.8 GB)
  BLS12-381 2^10     oracle/plonk.py 8 s
  BLS12-381 2^20     key build 68 s, reference at tau 12 s, key vs oracle/c 37 s, proof 0.8 s (8.2 GB),
                     reference checks 26 s
  BLS12-381 2^18 Rep3  key build 19 s, three-party proof 4 s (12.8 GB)
  BLS12-381 2^16 Shamir(3, 1)  key build 5 s, three-party proof 3 s (7.5 GB)
oracle/c's prover took 38 s at 2^20; at 2^22 it would add minutes to a case that is already the slowest of the file, so
the 2^22 proof is pinned by the trapdoor identities alone.
"""
import operator
import random
import threading
import time

import numpy as np
import pytest

from co_snarks_b200 import binding as B
from helpers import Conv, plonk_proof_from_device
from kernel_checks import bitrev_index
from oracle import plonk as OP
from oracle.ec import g1 as og1
from oracle.fields import CURVES, groth16_roots_of_unity
from workloads.synth_plonk import SELECTORS, SynthPlonk

CURVE_NAMES = ["bn254", "bls12_381"]


# ---------------------------------------------------------------------------------------------------- the reference
def _batch_inv(vals, r):
    pref = [1] * (len(vals) + 1)
    acc = 1
    for i, v in enumerate(vals):
        acc = acc * v % r
        pref[i + 1] = acc
    inv = pow(acc, r - 2, r)
    out = [0] * len(vals)
    for i in range(len(vals) - 1, -1, -1):
        out[i] = pref[i] * inv % r
        inv = inv * vals[i] % r
    return out


def _dot(x, y, r):
    return sum(map(operator.mul, x, y)) % r


class Barycentric:
    """L_i(x) = c u_i with c = (x^n - 1) / n and u_i = w^i / (x - w^i), for one x not in H."""

    def __init__(self, syn, x):
        r, n = syn.r, syn.n
        self.r, self.x = r, x
        self.xn = pow(x, n, r)
        self.zh = (self.xn - 1) % r
        assert self.zh, "x lies in H"
        self.c = self.zh * pow(n, r - 2, r) % r
        self.u = [w * v % r for w, v in zip(syn.omega, _batch_inv([(x - w) % r for w in syn.omega], r))]

    def at(self, values):
        """the polynomial with these values on H, at x"""
        return self.c * _dot(values, self.u, self.r) % self.r

    def lagrange(self, i):
        return self.c * self.u[i] % self.r


def wires_for(syn, full_witness):
    """The a, b, c wire values of every row for a full witness (leading one, public, private), additions included."""
    r, npub = syn.r, syn.n_public
    val = [0] + [int(x) % r for x in full_witness[1:]]
    for x, y, f1, f2 in syn.adds:
        val.append((val[x] * f1 + val[y] * f2) % r)
    pad = [0] * (syn.n - syn.n_constraints)
    assert npub < len(val)
    return tuple([val[s] for s in syn.key[m].tolist()] + pad for m in ("map_a", "map_b", "map_c"))


def sigma_values(syn):
    r, n = syn.r, syn.n
    coset = (1, syn.k1, syn.k2)
    pos = syn.sigma_pos.tolist()
    om = syn.omega
    return [[coset[p // n] * om[p % n] % r for p in pos[col * n:(col + 1) * n]] for col in range(3)]


class Reference:
    """The blinder- and challenge-independent part at tau for one synthetic key and full witness."""

    def __init__(self, syn, full_witness=None):
        self.syn, self.r, self.n = syn, syn.r, syn.n
        w = syn.full_witness if full_witness is None else full_witness
        self.pub = [int(x) % syn.r for x in w[1:syn.n_public + 1]]
        self.wires = wires_for(syn, w)
        self.sigma = sigma_values(syn)
        self.tau = syn.tau
        self.bt = Barycentric(syn, syn.tau)
        self.q_tau = [self.bt.at(s) for s in syn.selectors]
        self.s_tau = [self.bt.at(s) for s in self.sigma]
        self.w_tau = [self.bt.at(x) for x in self.wires]
        self.cd = CURVES[syn.curve]
        self.G = og1(self.cd)

    def g(self, k):
        return self.G.mul(self.cd.g1, k % self.r)

    def vk_points(self):
        return [self.g(x) for x in self.q_tau + self.s_tau]


def check_vk(ref, vk):
    exp = ref.vk_points()
    for i, k in enumerate(SELECTORS + ("s1", "s2", "s3")):
        assert vk[k] == exp[i], "verification key point %s != %s(tau) G1" % (k, k)


def check_proof(ref, proof, blinders):
    """Every trapdoor identity for `proof` (oracle dict) and the 11 blinders; raises AssertionError naming the first
    that fails.  -> the scalars it derived (challenges, polynomial values at tau)."""
    syn, r, n = ref.syn, ref.r, ref.n
    b = [int(x) % r for x in blinders]
    G, add, g = ref.G, ref.G.add, ref.g
    smul = lambda P, k: G.mul(P, k % r)
    tau, zh = ref.tau, ref.bt.zh
    k1, k2 = syn.k1, syn.k2
    vk = syn.vk_ints()
    out = {}
    # ---- round 1: wires
    blind1 = lambda x, lo, hi: (lo * x + hi)
    for i, k in enumerate("abc"):
        out[k] = (ref.w_tau[i] + blind1(tau, b[2 * i], b[2 * i + 1]) * zh) % r
        assert proof[k] == g(out[k]), "[%s] != %s(tau) G1" % (k.upper(), k)
    # ---- round 2: grand product
    t = OP.Transcript(ref.cd)
    for k in SELECTORS + ("s1", "s2", "s3"):
        t.add_point(vk[k])
    for v in ref.pub:
        t.add_scalar(v)
    for k in "abc":
        t.add_point(proof[k])
    beta = t.get_challenge()
    t = OP.Transcript(ref.cd)
    t.add_scalar(beta)
    gamma = t.get_challenge()
    A, Bw, Cw = ref.wires
    S1, S2, S3 = ref.sigma
    num, den = [], []
    for i, w in enumerate(syn.omega):
        bw = beta * w
        num.append((A[i] + bw + gamma) * (Bw[i] + k1 * bw + gamma) % r * (Cw[i] + k2 * bw + gamma) % r)
        den.append((A[i] + beta * S1[i] + gamma) * (Bw[i] + beta * S2[i] + gamma) % r * (Cw[i] + beta * S3[i] + gamma) % r)
    pn, pd, acc_n, acc_d = [], [], 1, 1
    for x, y in zip(num, den):
        acc_n, acc_d = acc_n * x % r, acc_d * y % r
        pn.append(acc_n)
        pd.append(acc_d)
    zb = [x * y % r for x, y in zip(pn, _batch_inv(pd, r))]
    zb = zb[-1:] + zb[:-1]  # Z_0 = the full product (1 for a witness that respects the copy constraints)
    zs = zb[1:] + zb[:1]    # values of z(w X) on H
    zbl = lambda x: (b[6] * x * x + b[7] * x + b[8]) % r
    out["z"] = z_tau = (ref.bt.at(zb) + zbl(tau) * zh) % r
    assert proof["z"] == g(z_tau), "[Z] != z(tau) G1"
    # ---- round 3: the quotient at tau
    t = OP.Transcript(ref.cd)
    t.add_scalar(beta)
    t.add_scalar(gamma)
    t.add_point(proof["z"])
    alpha = t.get_challenge()
    w_n = syn.omega[1] if n > 1 else 1
    zw_tau = (ref.bt.at(zs) + zbl(w_n * tau % r) * zh) % r
    a_, b_, c_ = out["a"], out["b"], out["c"]
    qm, ql, qr, qo, qc = ref.q_tau
    s1, s2, s3 = ref.s_tau
    pi = -sum(A[j] * ref.bt.lagrange(j) for j in range(max(1, syn.n_public)))
    gate = qm * a_ * b_ + ql * a_ + qr * b_ + qo * c_ + qc + pi
    bt = beta * tau
    perm = ((a_ + bt + gamma) * (b_ + k1 * bt + gamma) % r * (c_ + k2 * bt + gamma) % r * z_tau
            - (a_ + beta * s1 + gamma) * (b_ + beta * s2 + gamma) % r * (c_ + beta * s3 + gamma) % r * zw_tau)
    ident = (gate + alpha * perm + alpha * alpha % r * (z_tau - 1) % r * ref.bt.lagrange(0)) % r
    out["t"] = t_tau = ident * pow(zh, r - 2, r) % r
    tn = ref.bt.xn
    assert add(add(proof["t1"], smul(proof["t2"], tn)), smul(proof["t3"], tn * tn)) == g(t_tau), \
        "T sum: [T1] + tau^n [T2] + tau^2n [T3] != t(tau) G1"
    # ---- round 4: evaluations
    t = OP.Transcript(ref.cd)
    t.add_scalar(alpha)
    for k in ("t1", "t2", "t3"):
        t.add_point(proof[k])
    xi = t.get_challenge()
    bx = Barycentric(syn, xi)
    xiw = xi * w_n % r
    ev = {"eval_" + k: (bx.at(ref.wires[i]) + blind1(xi, b[2 * i], b[2 * i + 1]) * bx.zh) % r for i, k in enumerate("abc")}
    ev["eval_s1"], ev["eval_s2"] = bx.at(S1), bx.at(S2)
    ev["eval_zw"] = (bx.at(zs) + zbl(xiw) * bx.zh) % r
    for k, v in ev.items():
        assert proof[k] == v, "%s != the polynomial at xi" % k
    # ---- round 5: openings
    t = OP.Transcript(ref.cd)
    for x in (xi, ev["eval_a"], ev["eval_b"], ev["eval_c"], ev["eval_s1"], ev["eval_s2"], ev["eval_zw"]):
        t.add_scalar(x)
    v = [t.get_challenge()]
    for _ in range(4):
        v.append(v[-1] * v[0] % r)
    ea, eb, ec, es1, es2, ezw = (ev["eval_" + k] for k in ("a", "b", "c", "s1", "s2", "zw"))
    eval_pi = -sum(x * bx.lagrange(j) for j, x in enumerate(ref.pub))
    bxi = beta * xi
    e2 = (ea + bxi + gamma) * (eb + bxi * k1 + gamma) % r * (ec + bxi * k2 + gamma) % r * alpha % r
    e3 = (ea + beta * es1 + gamma) * (eb + beta * es2 + gamma) % r * ezw % r * alpha % r
    e4 = alpha * alpha % r * bx.lagrange(0) % r
    r0 = eval_pi - e3 * (ec + gamma) - e4
    S = (qm * (ea * eb % r) + ql * ea + qr * eb + qo * ec + qc - s3 * (e3 * beta % r) + z_tau * (e2 + e4) + r0
         + v[0] * (a_ - ea) + v[1] * (b_ - eb) + v[2] * (c_ - ec) + v[3] * (s1 - es1) + v[4] * (s2 - es2)) % r
    out["S"] = S
    t_xi = add(add(proof["t1"], smul(proof["t2"], bx.xn)), smul(proof["t3"], bx.xn * bx.xn))
    assert smul(proof["wxi"], tau - xi) == add(g(S), G.neg(smul(t_xi, bx.zh))), \
        "(tau - xi) [W_xi] != S G1 - Z_H(xi) ([T1] + xi^n [T2] + xi^2n [T3])"
    out["wxiw"] = (z_tau - ezw) * pow((tau - xiw) % r, r - 2, r) % r
    assert proof["wxiw"] == g(out["wxiw"]), "[W_xiw] != (z(tau) - z(xi w)) / (tau - xi w) G1"
    out.update(beta=beta, gamma=gamma, alpha=alpha, xi=xi, v=v)
    return out


def check_key(syn, n_ptau_samples=64, seed=7):
    """The key against references independent of the device: q / sigma / Lagrange coefficients and 4n-point
    evaluations against oracle/c's NTT, p_tau at its ends and at random indices against oracle.ec."""
    from oracle.c import run as OC
    cv, lg, n = Conv(syn.curve), syn.log_n, syn.n
    gm, gm4 = cv.fr([groth16_roots_of_unity(syn.r, lg)[0]]), cv.fr([groth16_roots_of_unity(syn.r, lg + 2)[0]])
    perm, perm4 = bitrev_index(lg).astype(np.int64), bitrev_index(lg + 2).astype(np.int64)
    key = syn.key

    def same(got, exp, what):
        if not np.array_equal(got, exp):
            bad = np.nonzero((got != exp).any(axis=1))[0]
            raise AssertionError("%s: %d of %d elements differ, first at %s" % (what, bad.size, len(exp), bad[:4].tolist()))

    def check(values_limbs, coeffs, evals4, what):
        co = OC.ifft_in_to_out(np.ascontiguousarray(values_limbs, dtype=np.uint64).copy(), lg, 1, gm, cv.id)[perm]
        if coeffs is not None:
            same(coeffs, co, what + " coefficients")
        ext = np.zeros((4 * n, 4), dtype=np.uint64)
        ext[:n] = co
        same(evals4, OC.fft_out_to_in(np.ascontiguousarray(ext[perm4]), lg + 2, 1, gm4, cv.id), what + " 4n evaluations")
    for k in range(5):
        check(cv.fr(syn.selectors[k]), key["q_coeffs"][k], key["q_evals"][k], SELECTORS[k])
    for col, vals in enumerate(sigma_values(syn)):
        check(cv.fr(vals), key["s_coeffs"][col], key["s_evals"][col], "s%d" % (col + 1))
    n4 = 4 * n
    for j in range(max(1, syn.n_public)):
        e = np.zeros((n, 4), dtype=np.uint64)
        e[j] = cv.fr([1])[0]
        check(e, None, key["lagrange_evals"][j * n4:(j + 1) * n4], "L_%d" % j)
    pts = key["p_tau"]
    m = pts.shape[0]
    assert m >= n + 6  # the blinded polynomials have n + 6 coefficients at most
    idx = sorted({0, m - 1} | set(random.Random(seed).sample(range(m), min(m, n_ptau_samples))))
    G, cd = og1(cv.c), cv.c
    for i in idx:
        assert cv.pt1(pts[i]) == G.mul(cd.g1, pow(syn.tau, i, syn.r)), "p_tau[%d] != tau^%d G1" % (i, i)


def verifier(curve):
    if curve == "bn254":
        from oracle.pairing_bn254 import pairing_product_is_one
    else:
        from oracle.pairing_bls12_381 import pairing_product_is_one
    return lambda syn, proof, pub: OP.verify(CURVES[curve], syn.vk_ints(), proof, pub, pairing_product_is_one)


def device_proof(syn, pk, bl):
    cv = Conv(syn.curve)
    return plonk_proof_from_device(cv, *pk.prove_plain(syn.public_inputs, syn.private_witness, cv.fr(bl)))


def _blinders(r, seed):
    rng = random.Random(seed)
    return [rng.randrange(r) for _ in range(11)]


# ---------------------------------------------------------------------------------------------------- MPC parties
def _threads(fn, n, timeout=1800):
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
        t.join(timeout=timeout)
    assert not errs, errs


def rep3_prove(mk, syn, bl, seed=23):
    """cs_plonk_rep3_prove with three party threads in peer mode (each its own context, key and session) on replicated
    shares of the private witness and of `bl`.  -> the three opened proofs."""
    cv, r = Conv(syn.curve), syn.r
    rng = random.Random(seed)

    def share(vals):
        out = [[], [], []]
        for v in vals:
            s0, s1 = rng.randrange(r), rng.randrange(r)
            sh = [s0, s1, (v - s0 - s1) % r]
            for p in range(3):
                out[p] += [sh[p], sh[(p + 2) % 3]]  # party p holds (x_p, x_{p-1})
        return [cv.fr(o).reshape(-1, 2, 4) for o in out]
    wsh, bsh = share(syn.full_witness[syn.n_public + 1:]), share(bl)
    ctxs = [mk() for _ in range(3)]
    pks, sess, nets, states = [], [], [], []
    try:
        pks = [B.PlonkKey(c, syn.cid, syn.key) for c in ctxs]
        sess = [B.PlonkRep3Session(ctxs[p], pks[p], p) for p in range(3)]
        nets = [B.Net.peer(ctxs[p], p, 3) for p in range(3)]
        for x in nets:
            x.connect_local(nets)
        for p in range(3):
            sess[p].connect(sess[(p + 1) % 3].arena)
            sess[p].connect_io(sess[(p + 2) % 3].d_out, sess[(p + 1) % 3].d_out)
        seeds = [bytes((31 * p + i) & 0xff for i in range(32)) for p in range(3)]
        states = [B.Rep3StateC.from_seeds(ctxs[0].lib, p, seeds[p], seeds[(p + 2) % 3]) for p in range(3)]
        res = {}

        def party(p):
            res[p] = sess[p].prove(nets[p], states[p], syn.public_inputs, wsh[p], bsh[p])
        _threads(party, 3)
        return [plonk_proof_from_device(cv, *res[p]) for p in range(3)]
    finally:
        for x in sess + pks + nets + states:
            x.free()
        for c in ctxs:
            c.close()


def _lagrange_at_zero(points, r):
    out = []
    for i in points:
        num, den = 1, 1
        for j in points:
            if j != i:
                num, den = num * j % r, den * (j - i) % r
        out.append(num * pow(den, r - 2, r) % r)
    return out


def shamir_prove(mk, syn, n=3, t=1, seed=5):
    """cs_plonk_shamir_prove with n party threads on degree-t shares of the private witness; the parties draw the
    blinders.  -> (opened proofs, the blinders reconstructed from parties 0..t and from parties n-t-1..n-1)."""
    cv, r = Conv(syn.curve), syn.r
    rng = random.Random(seed)
    wsh = [[] for _ in range(n)]
    for v in syn.full_witness[syn.n_public + 1:]:
        co = [v] + [rng.randrange(r) for _ in range(t)]
        for i in range(n):
            wsh[i].append(sum(c * pow(i + 1, k, r) for k, c in enumerate(co)) % r)
    ctxs = [mk() for _ in range(n)]
    pks, sess, nets = [], [], []
    try:
        pks = [B.PlonkKey(c, syn.cid, syn.key) for c in ctxs]
        sess = [B.PlonkShamirSession(ctxs[p], pks[p], n, t, p) for p in range(n)]
        nets = [B.Net.peer(ctxs[i], i, n) for i in range(n)]
        for x in nets:
            x.connect_local(nets)
        res = {}

        def party(p):
            res[p] = sess[p].prove(nets[p], syn.public_inputs, cv.fr(wsh[p]))
        _threads(party, n)
        proofs = [plonk_proof_from_device(cv, *res[p][:2]) for p in range(n)]
        sh = [cv.fr_back(res[p][2]) for p in range(n)]

        def rec(subset):
            lam = _lagrange_at_zero([p + 1 for p in subset], r)
            return [sum(l * sh[p][i] for l, p in zip(lam, subset)) % r for i in range(11)]
        return proofs, rec(list(range(t + 1))), rec(list(range(n - t - 1, n)))
    finally:
        for x in sess + pks + nets:
            x.free()
        for c in ctxs:
            c.close()


# ---------------------------------------------------------------------------------------------------- CPU (emulation)
def _emu_factory():
    import os
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
    import build_emu
    path = build_emu.build()
    return lambda: B.Context(0, lib_path=path)


def test_default_synth_plonk_unchanged_emu(emu_ctx):
    """SynthPlonk(ctx, lg) with default arguments is the circuit the co-Plonk timing tool and the benchmark prove: its
    BN254 key and witness at 2^8 hash to the value taken before the curve and gate options existed."""
    import hashlib
    syn = SynthPlonk(emu_ctx, 8)
    h = hashlib.sha256()
    for name in sorted(syn.key):
        v = syn.key[name]
        for a in (v if isinstance(v, list) else [v]):
            h.update(name.encode())
            h.update(np.ascontiguousarray(a).tobytes() if isinstance(a, np.ndarray) else str(a).encode())
    h.update(np.ascontiguousarray(syn.public_inputs).tobytes())
    h.update(np.ascontiguousarray(syn.private_witness).tobytes())
    assert h.hexdigest() == "73b9b2fbe235dcfcc782b2373c564532d76c20060722950f4911280661501f62"


@pytest.mark.parametrize("curve", CURVE_NAMES)
@pytest.mark.parametrize("gates", ["fixed", "mixed"])
def test_reference_equals_oracle_emu(emu_ctx, curve, gates):
    """At 2^6 with 5 public inputs the reference's values equal oracle/plonk.py's polynomials at tau, element by
    element, and oracle/plonk.py's proof satisfies every identity."""
    syn = SynthPlonk(emu_ctx, 6, n_public=5, curve=curve, gates=gates)
    r, tau = syn.r, syn.tau
    ref = Reference(syn)
    assert ref.wires == syn.wires
    if gates == "mixed":
        assert all(any(v not in (0, 1, r - 1, 5) for v in s) for s in syn.selectors)
        assert any(syn.selectors[0][i] == 0 and syn.selectors[3][i] for i in range(syn.n))
        assert any(syn.selectors[1][i] == syn.selectors[2][i] == 0 and syn.selectors[0][i] for i in range(syn.n))
    z = syn.oracle_zkey()
    check_vk(ref, syn.vk_ints())
    bl = _blinders(r, 3)
    trace = {}
    proof = OP.prove(z, syn.full_witness, bl, trace=trace)
    got = check_proof(ref, proof, bl)
    ev = lambda p, x=tau: OP._eval(p, x, r)
    for k in ("a", "b", "c", "z"):
        assert got[k] == ev(trace["polys"][k]), k
    tn = pow(tau, syn.n, r)
    assert got["t"] == (ev(trace["t1"]) + tn * ev(trace["t2"]) + tn * tn * ev(trace["t3"])) % r
    assert got["wxiw"] == ev(trace["wxiw"])
    xi = got["xi"]
    xn = pow(xi, syn.n, r)
    assert (tau - xi) * ev(trace["wxi"]) % r == (got["S"] - (xn - 1) * (ev(trace["t1"]) + xn * ev(trace["t2"]) + xn * xn * ev(trace["t3"]))) % r
    for k in ("beta", "gamma", "alpha", "xi", "v"):
        assert got[k] == trace[k], k


@pytest.mark.parametrize("curve", CURVE_NAMES)
@pytest.mark.parametrize("gates", ["fixed", "mixed"])
def test_device_proof_emu(emu_ctx, curve, gates):
    """The emulated device proof at 2^7 satisfies every identity, equals oracle/plonk.py's and verifies; the key passes
    the oracle/c NTT and p_tau checks."""
    syn = SynthPlonk(emu_ctx, 7, n_public=4, curve=curve, gates=gates)
    ref = Reference(syn)
    check_key(syn)
    check_vk(ref, syn.vk_ints())
    pk = syn.make_key()
    bl = _blinders(syn.r, 11)
    proof = device_proof(syn, pk, bl)
    pk.free()
    check_proof(ref, proof, bl)
    assert proof == OP.prove(syn.oracle_zkey(), syn.full_witness, bl)
    assert verifier(curve)(syn, proof, ref.pub)


@pytest.mark.parametrize("curve", CURVE_NAMES)
def test_changed_witness_fails_t_sum_emu(emu_ctx, curve):
    """Negative control: with the last private value changed (its gate no longer holds, the copy constraints still do)
    the device proof passes the A, B, C and Z checks, fails the T sum, and the verifier rejects it."""
    syn = SynthPlonk(emu_ctx, 6, curve=curve, gates="mixed")
    w = list(syn.full_witness)
    w[-1] = (w[-1] + 1) % syn.r
    ref = Reference(syn, w)
    pk = syn.make_key()
    bl = _blinders(syn.r, 13)
    cv = Conv(curve)
    proof = plonk_proof_from_device(cv, *pk.prove_plain(syn.public_inputs, cv.fr(w[syn.n_public + 1:]), cv.fr(bl)))
    pk.free()
    with pytest.raises(AssertionError, match="T sum"):
        check_proof(ref, proof, bl)
    assert not verifier(curve)(syn, proof, ref.pub)


@pytest.mark.parametrize("curve", CURVE_NAMES)
def test_b9_gap_emu(emu_ctx, curve):
    """Negative control: b9 moves a multiple of X^n between T1 and T2, which the T sum, the opening identities and the
    verifier cannot see.  With b9 off by one on the reference side only, exact equality with oracle/plonk.py fails while
    the trapdoor identities and the verifier still accept the device proof."""
    syn = SynthPlonk(emu_ctx, 6, curve=curve, gates="mixed")
    ref = Reference(syn)
    pk = syn.make_key()
    bl = _blinders(syn.r, 17)
    proof = device_proof(syn, pk, bl)
    pk.free()
    z = syn.oracle_zkey()
    assert proof == OP.prove(z, syn.full_witness, bl)
    off = list(bl)
    off[9] = (off[9] + 1) % syn.r
    assert proof != OP.prove(z, syn.full_witness, off)
    check_proof(ref, proof, off)
    assert verifier(curve)(syn, proof, ref.pub)


def test_rep3_peer_bls12_381_emu(emu_ctx):
    """Rep3 (in-library driver, peer mode) at 2^6 on BLS12-381, mixed gates: all parties open the same proof, it equals
    the plain proof for the summed blinders and satisfies the reference."""
    syn = SynthPlonk(emu_ctx, 6, n_public=4, curve="bls12_381", gates="mixed")
    bl = _blinders(syn.r, 19)
    proofs = rep3_prove(_emu_factory(), syn, bl)
    assert proofs[0] == proofs[1] == proofs[2], "parties disagree on the proof"
    pk = syn.make_key()
    assert proofs[0] == device_proof(syn, pk, bl)
    pk.free()
    check_proof(Reference(syn), proofs[0], bl)


def test_shamir_bls12_381_emu(emu_ctx):
    """Shamir(3, 1) at 2^6 on BLS12-381, mixed gates, blinders drawn by the parties: the opened proof satisfies the
    reference for the blinders the shares reconstruct to."""
    syn = SynthPlonk(emu_ctx, 6, n_public=4, curve="bls12_381", gates="mixed")
    proofs, bl, bl2 = shamir_prove(_emu_factory(), syn)
    assert all(p == proofs[0] for p in proofs), "parties disagree on the proof"
    assert bl == bl2 and len(set(bl)) == 11
    check_proof(Reference(syn), proofs[0], bl)


# ---------------------------------------------------------------------------------------------------- GPU
class Peak:
    """Wall time and the peak of (total - free) device memory while the block runs, sampled every 20 ms."""

    def __init__(self, what):
        self.what = what

    def __enter__(self):
        import torch
        self.info = lambda: (lambda f, t: t - f)(*torch.cuda.mem_get_info(0))
        self.base = self.peak = self.info()
        self.stop = threading.Event()

        def poll():
            while not self.stop.wait(0.02):
                self.peak = max(self.peak, self.info())
        self.th = threading.Thread(target=poll, daemon=True)
        self.th.start()
        self.t0 = time.time()
        return self

    def __exit__(self, *exc):
        self.stop.set()
        self.th.join()
        print("\n[plonk-trapdoor] %s: %.1f s, peak %.2f GB used (%.2f GB at start)"
              % (self.what, time.time() - self.t0, self.peak / 1e9, self.base / 1e9))


def _gpu_factory():
    return lambda: B.Context(0)


def _syn_fixture(ctx, lg, **kw):
    with Peak("key 2^%d %s" % (lg, kw)):
        syn = SynthPlonk(ctx, lg, **kw)
    with Peak("reference at tau 2^%d" % lg):
        ref = Reference(syn)
    return syn, ref


def _free(syn):
    syn.key = None


@pytest.fixture(scope="class")
def bn254_2p20_mixed(gpu_ctx):
    syn, ref = _syn_fixture(gpu_ctx, 20, n_public=4, gates="mixed")
    yield syn, ref
    _free(syn)


@pytest.fixture(scope="class")
def bn254_2p22(gpu_ctx):
    syn, ref = _syn_fixture(gpu_ctx, 22)
    yield syn, ref
    _free(syn)


@pytest.fixture(scope="class")
def bls_2p20_mixed(gpu_ctx):
    syn, ref = _syn_fixture(gpu_ctx, 20, n_public=4, curve="bls12_381", gates="mixed")
    yield syn, ref
    _free(syn)


def _plain_case(syn, ref, what, seed):
    check_vk(ref, syn.vk_ints())
    bl = _blinders(syn.r, seed)
    with Peak("plain proof " + what):
        pk = syn.make_key()
        proof = device_proof(syn, pk, bl)
        pk.free()
    with Peak("reference checks " + what):
        check_proof(ref, proof, bl)
    return proof, bl


@pytest.mark.gpu
class TestBn254Mixed2p20:
    @pytest.fixture
    def key(self, bn254_2p20_mixed):
        return bn254_2p20_mixed

    def test_key(self, key):
        with Peak("key checks bn254 2^20"):
            check_key(key[0])

    def test_proof_equals_oracle_c(self, key):
        from oracle.c import run as OC
        syn, ref = key
        proof, bl = _plain_case(syn, ref, "bn254 2^20 mixed", 21)
        with Peak("oracle/c plonk_prove bn254 2^20"):
            pts, evs = OC.plonk_prove(syn.key, syn.public_inputs, syn.private_witness, syn.fr(bl))
        assert plonk_proof_from_device(Conv("bn254"), pts, evs) == proof


@pytest.mark.gpu
class TestBn254Configs3:
    """The domain and circuit of BASELINE configs[3] (the default synthetic circuit at 2^22), plain."""

    @pytest.fixture
    def key(self, bn254_2p22):
        return bn254_2p22

    def test_key(self, key):
        with Peak("key checks bn254 2^22"):
            check_key(key[0])

    def test_plain(self, key):
        _plain_case(*key, "bn254 2^22", 23)


@pytest.mark.gpu
def test_rep3_peer_bn254_2p21_gpu(gpu_ctx):
    """Rep3 on the configs[3] circuit, one size below its domain: three parties at 2^21 already peak at 73 GB of an
    80 GB card, and one plain 2^22 proof alone at 22 GB, so three party keys and sessions at 2^22 do not fit."""
    syn, ref = _syn_fixture(gpu_ctx, 21)
    bl = _blinders(syn.r, 29)
    with Peak("rep3 peer bn254 2^21"):
        proofs = rep3_prove(_gpu_factory(), syn, bl)
    assert proofs[0] == proofs[1] == proofs[2], "parties disagree on the proof"
    pk = syn.make_key()
    plain = device_proof(syn, pk, bl)
    pk.free()
    assert proofs[0] == plain, "opened Rep3 proof != plain proof for the summed blinders"
    check_proof(ref, proofs[0], bl)


@pytest.mark.gpu
def test_bls12_381_2p10_equals_oracle_gpu(gpu_ctx):
    syn = SynthPlonk(gpu_ctx, 10, n_public=4, curve="bls12_381", gates="mixed")
    ref = Reference(syn)
    check_key(syn)
    proof, bl = _plain_case(syn, ref, "bls12_381 2^10 mixed", 31)
    with Peak("oracle/plonk.py bls12_381 2^10"):
        assert proof == OP.prove(syn.oracle_zkey(), syn.full_witness, bl)


@pytest.mark.gpu
class TestBls12381Mixed2p20:
    @pytest.fixture
    def key(self, bls_2p20_mixed):
        return bls_2p20_mixed

    def test_key(self, key):
        with Peak("key checks bls12_381 2^20"):
            check_key(key[0])

    def test_plain(self, key):
        _plain_case(*key, "bls12_381 2^20 mixed", 37)


@pytest.mark.gpu
def test_rep3_peer_bls12_381_2p18_gpu(gpu_ctx):
    syn, ref = _syn_fixture(gpu_ctx, 18, n_public=4, curve="bls12_381", gates="mixed")
    check_key(syn)
    bl = _blinders(syn.r, 41)
    with Peak("rep3 peer bls12_381 2^18"):
        proofs = rep3_prove(_gpu_factory(), syn, bl)
    assert proofs[0] == proofs[1] == proofs[2], "parties disagree on the proof"
    pk = syn.make_key()
    assert proofs[0] == device_proof(syn, pk, bl), "opened Rep3 proof != plain proof for the summed blinders"
    pk.free()
    check_proof(ref, proofs[0], bl)


@pytest.mark.gpu
def test_shamir_bls12_381_2p16_gpu(gpu_ctx):
    syn, ref = _syn_fixture(gpu_ctx, 16, n_public=4, curve="bls12_381", gates="mixed")
    check_key(syn)
    with Peak("shamir(3, 1) bls12_381 2^16"):
        proofs, bl, bl2 = shamir_prove(_gpu_factory(), syn)
    assert all(p == proofs[0] for p in proofs), "parties disagree on the proof"
    assert bl == bl2
    check_proof(ref, proofs[0], bl)
