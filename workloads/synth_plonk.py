"""Synthetic Plonk workload of any size with a VALID snarkjs-style proving key (known tau), for the full-size
tests and the Plonk timing tool (BASELINE.json configs[3] names a synthetic Plonk circuit; SURVEY.md 8d).

Not part of the product path and not the oracle: it only manufactures inputs.  The reference has no setup
code (keys come from snarkjs); what is built here follows the snarkjs Plonk arithmetisation the prover
assumes (co-plonk/src/round2.rs:99-160, round3.rs:330-420): gate  qm a b + ql a + qr b + qo c + qc + PI = 0
with PI(X) = -sum_j w_pub[j] L_j(X), one `ql = 1` row per public input, copy constraints through
sigma_1..3 over the cosets H, k1 H, k2 H, and "additions" (linear combinations of earlier signals that are not
part of the witness, round1.rs:191-224).  A key built here is accepted by the oracle's verifier
(oracle/plonk.py, itself pinned on the reference's fixtures), which is what makes large proofs checkable.

Circuit (seeded): signal 0 is the constant slot (value 0 in Plonk), 1..n_public public, then private signals,
then additions.  Row i < n_public exposes public signal i + 1.  Every later row defines a new private signal
c from two earlier signals; every 16th row first defines an addition s = f1 x + f2 y and uses it as the b wire.
Three rows at the end are left empty (all-zero selectors, wires on signal 0).  With gates="fixed" (the default,
what the timing tools use) every row is c = a b + a + 5 (qm = 1, ql = 1, qo = -1, qc = 5).  With gates="mixed"
every row draws full-width qm, ql, qr, qc and a nonzero qo and solves for c; every third row is linear (qm = 0)
and every third row has ql = qr = 0, so each selector takes arbitrary values and q_R is not identically zero.

Keys are built for BN254 (the default) or BLS12-381 (`curve`).  What an exact reference of the proof needs is kept
on the object: `tau`, `omega` (the powers of the domain generator), `selectors` (qm, ql, qr, qo, qc as values on
H), `sigma_pos` (the permutation: position p of column p // n, row p % n maps to position sigma_pos[p]) and
`wires` (the a, b, c values per row).
"""
import random

import numpy as np

from co_snarks_b200 import binding as B
from oracle.fields import CURVES

BN254_R = 21888242871839275222246405745257275088548364400416034343698204186575808495617
BN254_Q = 21888242871839275222246405745257275088696311157297823662689037894645226208583
CURVE_IDS = {"bn254": B.CS_BN254, "bls12_381": B.CS_BLS12_381}
SELECTORS = ("qm", "ql", "qr", "qo", "qc")


def _fr(vals, r=BN254_R):
    return B.ints_to_limbs(B.to_mont_ints(vals, r, 4), 4)


class SynthPlonk:
    def __init__(self, ctx, log_n, seed=1, setup_seed=2, n_public=2, add_every=16, curve="bn254", gates="fixed"):
        assert gates in ("fixed", "mixed")
        cd = CURVES[curve]
        r, q, nq = cd.r, cd.q, cd.nq
        c = CURVE_IDS[curve]
        self.ctx, self.curve, self.cid, self.r, self.q, self.nq = ctx, curve, c, r, q, nq
        fr = lambda vals: _fr(vals, r)
        self.fr = fr
        self.n = n = 1 << log_n
        n4 = 4 * n
        rng = random.Random(seed)
        nc = n - 3
        k1, k2 = 2, 3
        gen, _ = ctx.roots_of_unity(c, log_n)
        w_n = B.from_mont_ints(B.limbs_to_ints(gen.reshape(1, 4)), r, 4)[0]
        assert pow(k1, n, r) != 1 and pow(k2, n, r) != 1 and pow(k2 * pow(k1, -1, r) % r, n, r) != 1
        # ---- circuit + assignment
        n_add = max(0, (nc - n_public) // add_every) if add_every else 0
        n_priv = nc - n_public
        first_add = 1 + n_public + n_priv
        n_vars = first_add + n_add
        val = [0] * n_vars  # Plonk's view: signal 0 reads as zero (types.rs:118-120)
        for i in range(1, n_public + 1):
            val[i] = rng.randrange(r)
        map_a, map_b, map_c = [0] * nc, [0] * nc, [0] * nc
        sel = np.zeros((5, n), dtype=np.int8)  # qm ql qr qo qc as small integers (-1 -> r - 1), gates="fixed"
        mixed = [[0] * n for _ in range(5)] if gates == "mixed" else None  # full-width values, gates="mixed"
        adds = []
        defined = list(range(0, n_public + 1))  # signal 0 reads as zero and may feed gates
        nxt = n_public + 1
        for i in range(n_public):
            map_a[i] = i + 1
            sel[1, i] = 1
            if mixed:
                mixed[1][i] = 1
        for i in range(n_public, nc):
            a = defined[rng.randrange(len(defined))]
            b = defined[rng.randrange(len(defined))]
            if add_every and (i - n_public) % add_every == add_every - 1 and len(adds) < n_add:
                x, y = defined[rng.randrange(len(defined))], defined[rng.randrange(len(defined))]
                f1, f2 = rng.randrange(1, r), rng.randrange(1, r)
                s = first_add + len(adds)
                adds.append((x, y, f1, f2))
                val[s] = (val[x] * f1 + val[y] * f2) % r
                defined.append(s)
                b = s
            cc = nxt
            nxt += 1
            if mixed:
                qm, ql, qr, qo, qc = (rng.randrange(r), rng.randrange(r), rng.randrange(r), rng.randrange(1, r),
                                      rng.randrange(r))
                if i % 3 == 1:
                    qm = 0
                elif i % 3 == 2:
                    ql = qr = 0
                for k, v in enumerate((qm, ql, qr, qo, qc)):
                    mixed[k][i] = v
                val[cc] = -(qm * val[a] * val[b] + ql * val[a] + qr * val[b] + qc) * pow(qo, -1, r) % r
            else:
                val[cc] = (val[a] * val[b] + val[a] + 5) % r
                sel[0, i], sel[1, i], sel[3, i], sel[4, i] = 1, 1, -1, 5
            defined.append(cc)
            map_a[i], map_b[i], map_c[i] = a, b, cc
        n_add = len(adds)
        n_vars = first_add + n_add
        assert nxt == first_add
        self.n_public, self.n_vars, self.n_additions, self.n_constraints = n_public, n_vars, n_add, nc
        self.full_witness = [1] + val[1:first_add]  # what a .wtns file holds (leading one, no additions)
        self.wires = tuple([val[s] for s in m] + [0] * (n - nc) for m in (map_a, map_b, map_c))
        if mixed:
            self.selectors = mixed
        else:
            small = {v: v % r for v in (0, 1, -1, 5)}
            self.selectors = [[small[int(v)] for v in sel[k]] for k in range(5)]
        # ---- selector / sigma / Lagrange polynomials: evaluations on H -> coefficients -> 4n evaluations (device NTTs)
        consts = {v: fr([v % r])[0] for v in (0, 1, -1, 5)}
        dom, dom4 = ctx.domain(c, log_n, gen), ctx.domain(c, log_n + 2, ctx.roots_of_unity(c, log_n + 2)[0])
        d_n, d_4n = ctx.alloc(n * 32), ctx.alloc(n4 * 32)

        def to_polys(evals_limbs):
            ctx.h2d(d_n, evals_limbs)
            dom.ifft(d_n)
            co = ctx.d2h(d_n, (n, 4))
            ext = np.zeros((n4, 4), dtype=np.uint64)
            ext[:n] = co
            ctx.h2d(d_4n, ext)
            dom4.fft(d_4n)
            return co, ctx.d2h(d_4n, (n4, 4))
        q_coeffs, q_evals = [], []
        for k in range(5):
            if mixed:
                ev = fr(mixed[k])
            else:
                ev = np.zeros((n, 4), dtype=np.uint64)
                for v, limbs in consts.items():
                    ev[sel[k] == v] = limbs
            co, e4 = to_polys(ev)
            q_coeffs.append(co)
            q_evals.append(e4)
        # identity values of the three cosets, then the permutation: each signal's positions form one cycle
        wi, omega = 1, []
        for _ in range(n):
            omega.append(wi)
            wi = wi * w_n % r
        ids = np.concatenate([fr(omega), fr([k1 * x % r for x in omega]), fr([k2 * x % r for x in omega])])
        sig = np.zeros(3 * n, dtype=np.int64)
        maps = np.zeros((3, n), dtype=np.int64)
        maps[0, :nc], maps[1, :nc], maps[2, :nc] = map_a, map_b, map_c
        flat = maps.reshape(-1)
        order = np.argsort(flat, kind="stable")  # positions grouped by signal
        grouped = flat[order]
        starts = np.flatnonzero(np.r_[True, grouped[1:] != grouped[:-1]])
        ends = np.r_[starts[1:], len(order)]
        nxt_pos = np.empty_like(order)
        nxt_pos[:-1] = order[1:]
        nxt_pos[ends - 1] = order[starts]  # close each cycle
        sig[order] = nxt_pos
        self.omega, self.sigma_pos = omega, sig
        s_coeffs, s_evals = [], []
        for col in range(3):
            co, e4 = to_polys(ids[sig[col * n:(col + 1) * n]])
            s_coeffs.append(co)
            s_evals.append(e4)
        nlag = max(1, n_public)
        lag = np.zeros((nlag * n4, 4), dtype=np.uint64)
        for j in range(nlag):
            ev = np.zeros((n, 4), dtype=np.uint64)
            ev[j] = consts[1]
            _, e4 = to_polys(ev)
            lag[j * n4:(j + 1) * n4] = e4
        ctx.free(d_n)
        ctx.free(d_4n)
        dom.free()
        dom4.free()
        # ---- SRS with known tau, commitments of the verification key
        srng = random.Random(setup_seed)
        self.tau = tau = srng.randrange(2, r)
        npt = n + 8
        pw, t = [], 1
        for _ in range(npt):
            pw.append(t)
            t = t * tau % r
        g1 = B.ints_to_limbs(B.to_mont_ints(list(cd.g1), q, nq), nq).reshape(-1)
        g2 = B.ints_to_limbs(B.to_mont_ints([cd.g2[0][0], cd.g2[0][1], cd.g2[1][0], cd.g2[1][1]], q, nq), nq).reshape(-1)
        p_tau = ctx.fixed_base_mul(c, B.CS_G1, g1, fr(pw))
        self.x2 = ctx.fixed_base_mul(c, B.CS_G2, g2, fr([tau]))[0]
        bases = ctx.bases_upload(c, B.CS_G1, p_tau)
        vk_points = np.stack([ctx.msm(bases, co, n=n, montgomery=True)[0] for co in q_coeffs + s_coeffs])
        bases.free()
        na = n_add
        self.key = dict(n_vars=n_vars, n_public=n_public, domain_size=n, n_additions=na, n_constraints=nc,
                        k1=fr([k1]), k2=fr([k2]), vk_points=vk_points,
                        additions_ids=np.array([[x, y] for x, y, _, _ in adds], dtype=np.uint32).reshape(na, 2),
                        additions_factors=fr([f for _, _, f1, f2 in adds for f in (f1, f2)]).reshape(na, 2, 4),
                        map_a=np.array(map_a, dtype=np.uint32), map_b=np.array(map_b, dtype=np.uint32),
                        map_c=np.array(map_c, dtype=np.uint32), q_coeffs=q_coeffs, q_evals=q_evals,
                        s_coeffs=s_coeffs, s_evals=s_evals, lagrange_evals=lag, p_tau=p_tau)
        self.k1, self.k2, self.log_n = k1, k2, log_n
        self.adds = adds
        self.public_inputs = fr(self.full_witness[:n_public + 1])
        self.private_witness = fr(self.full_witness[n_public + 1:])

    def make_key(self):
        return B.PlonkKey(self.ctx, self.cid, self.key)

    def _points(self, a):
        nq = self.nq
        v = B.from_mont_ints(B.limbs_to_ints(np.asarray(a).reshape(-1, nq)), self.q, nq)
        return [None if (v[2 * i] == 0 and v[2 * i + 1] == 0) else (v[2 * i], v[2 * i + 1]) for i in range(len(v) // 2)]

    def vk_ints(self):
        """Verification key in the oracle's conventions (oracle.plonk.verify)."""
        v = B.from_mont_ints(B.limbs_to_ints(np.asarray(self.x2).reshape(-1, self.nq)), self.q, self.nq)
        vk = dict(n_public=self.n_public, power=self.log_n, k1=self.k1, k2=self.k2, x2=((v[0], v[1]), (v[2], v[3])))
        pts = self._points(self.key["vk_points"])
        for i, k in enumerate(SELECTORS + ("s1", "s2", "s3")):
            vk[k] = pts[i]
        return vk

    def oracle_zkey(self):
        """The same key as python ints for oracle.plonk.prove (small sizes only)."""
        r = self.r
        back = lambda a: B.from_mont_ints(B.limbs_to_ints(a), r, 4)
        n4 = 4 * self.n
        z = dict(curve=CURVES[self.curve], q=self.q, r=r, n_vars=self.n_vars, n_public=self.n_public,
                 domain_size=self.n, n_additions=self.n_additions, n_constraints=self.n_constraints, k1=self.k1,
                 k2=self.k2, additions=list(self.adds), map_a=[int(x) for x in self.key["map_a"]],
                 map_b=[int(x) for x in self.key["map_b"]], map_c=[int(x) for x in self.key["map_c"]])
        vk = self.vk_ints()
        for i, k in enumerate(SELECTORS):
            z[k] = dict(coeffs=back(self.key["q_coeffs"][i]), evals=back(self.key["q_evals"][i]))
            z["vk_" + k] = vk[k]
        for i, k in enumerate(("s1", "s2", "s3")):
            z[k] = dict(coeffs=back(self.key["s_coeffs"][i]), evals=back(self.key["s_evals"][i]))
            z["vk_" + k] = vk[k]
        lag = self.key["lagrange_evals"]
        z["lagrange"] = [dict(coeffs=None, evals=back(lag[j * n4:(j + 1) * n4])) for j in range(max(1, self.n_public))]
        z["p_tau"] = self._points(self.key["p_tau"])
        z["x2"] = vk["x2"]
        return z
