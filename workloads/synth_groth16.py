"""Synthetic Groth16 workload of any size with a VALID proving key (known toxic waste), for bench.py
and the full-size tests.  BASELINE.json configs[1]/[2]: "synthetic R1CS 2^20 constraints".

Not part of the product path and not the oracle: it only manufactures inputs.  The reference has no
setup code (keys come from snarkjs); the formulas are SURVEY.md 8(d)'s derivation, and a key built
here is accepted by the same pairing check that accepts the reference's snarkjs fixtures
(tests/test_gpu_fullsize.py), which is what makes full-size proofs checkable.

R1CS (seeded): variables w[0] = 1, w[1] = public input, w[k] for k >= 2 defined by constraint
k - 2:  (w[j1] + w[j2]) * w[j3] = w[k]  with j1, j2, j3 < k   ->  2 nnz per A row, 1 per B row.
num_constraints = m - 2 (2^log_m - 2 unless given), num_instance_variables = 2, so domain = next_pow2(m)
(reduction.rs:85).  Keys are built for BN254 (the default) or BLS12-381; generators, moduli and roots of
unity (co-groth16/src/groth16.rs:60-100) come from oracle.fields.
Scalars for the query points are computed on the host with python ints; the 5 n fixed-base
multiplications run on the GPU through cs_fixed_base_mul.
"""
import random

import numpy as np

from co_snarks_b200 import binding as B
from oracle.fields import CURVES, groth16_roots_of_unity

BN254_R = 21888242871839275222246405745257275088548364400416034343698204186575808495617
BN254_Q = 21888242871839275222246405745257275088696311157297823662689037894645226208583
CURVE_IDS = {"bn254": B.CS_BN254, "bls12_381": B.CS_BLS12_381}


def _batch_inv(vals, p):
    n = len(vals)
    pref = [1] * (n + 1)
    for i, v in enumerate(vals):
        pref[i + 1] = pref[i] * v % p
    inv = pow(pref[n], p - 2, p)
    out = [0] * n
    for i in range(n - 1, -1, -1):
        out[i] = pref[i] * inv % p
        inv = inv * vals[i] % p
    return out


def _fr(vals, r=BN254_R):
    return B.ints_to_limbs(B.to_mont_ints(vals, r, 4), 4)


def _fq_pts(flat, k, q=BN254_Q, nq=4):
    return B.ints_to_limbs(B.to_mont_ints(flat, q, nq), nq).reshape(-1, nq * k)


def make_r1cs(m, seed=1, r=BN254_R):
    """-> (a_rows, b_rows, c_cols, witness): rows as lists of (coeff, var); witness = full assignment."""
    rng = random.Random(seed)
    w = [1, rng.randrange(r)]
    a_rows, b_rows, c_cols = [], [], []
    for k in range(2, m):
        j1, j2, j3 = rng.randrange(k), rng.randrange(k), rng.randrange(k)
        if j1 == j2:
            a_rows.append([(2, j1)])
        else:
            a_rows.append([(1, j1), (1, j2)])
        b_rows.append([(1, j3)])
        c_cols.append(k)
        w.append((w[j1] + w[j2]) * w[j3] % r)
    return a_rows, b_rows, c_cols, w


class SynthGroth16:
    """Builds matrices + key; `key_arrays` are what cs_groth16_pk_create consumes."""

    def __init__(self, ctx, log_m, seed=1, setup_seed=2, valid=True, r1cs=None, curve="bn254", num_constraints=None,
                 keep_trapdoor=False):
        """r1cs = (a_rows, b_rows, c_rows, full_witness, num_instance_variables) builds a key for an explicit
        system instead of the seeded chain (rows = lists of (coeff, variable)).  num_constraints sizes the seeded
        chain (default 2^log_m - 2).  keep_trapdoor=True keeps (tau, alpha, beta, gamma, delta) as `trapdoor` and the
        per-variable scalars u_i(tau), v_i(tau), w_i(tau) and the h_query scalars as `At`, `Bt`, `Ct`, `h_sc`."""
        cd = CURVES[curve]
        r, q = cd.r, cd.q
        self.ctx, self.curve, self.cid, self.r, self.q, self.nq = ctx, curve, CURVE_IDS[curve], r, q, cd.nq
        if r1cs is None:
            self.nc = (1 << log_m) - 2 if num_constraints is None else num_constraints
            self.m = m = self.nc + 2
            self.ni = 2
            log_m = max(0, (m - 1).bit_length())
            a_rows, b_rows, c_cols, self.witness = make_r1cs(m, seed, r)
            c_rows = [[(1, v)] for v in c_cols]
        else:
            a_rows, b_rows, c_rows, self.witness, self.ni = r1cs
            self.m = m = len(self.witness)
            self.nc = len(a_rows)
            log_m = max(0, (self.nc + self.ni - 1).bit_length())
        self.n = n = 1 << log_m  # domain size = next_power_of_two(nc + ni)
        self.a_rows, self.b_rows = a_rows, b_rows
        rng = random.Random(setup_seed)
        tau, alpha, beta, gamma, delta = (rng.randrange(1, r) for _ in range(5))
        if keep_trapdoor:
            assert valid, "an invalid key has no trapdoor"
            self.trapdoor = dict(tau=tau, alpha=alpha, beta=beta, gamma=gamma, delta=delta)
        # the roots are computed here rather than read from the library, so that a key is independent of the roots
        # and coset shift the library's witness map uses
        w_n, w_2n = groth16_roots_of_unity(r, log_m)
        if valid:
            # L_j(tau) = (tau^n - 1) w^j / (n (tau - w^j))
            zn = (pow(tau, n, r) - 1) % r
            wj, pw = 1, []
            for _ in range(n):
                pw.append(wj)
                wj = wj * w_n % r
            inv = _batch_inv([(n * (tau - x)) % r for x in pw], r)
            L = [zn * x % r * iv % r for x, iv in zip(pw, inv)]
            At, Bt, Ct = [0] * m, [0] * m, [0] * m
            for j, row in enumerate(a_rows):
                for cf, v in row:
                    At[v] = (At[v] + cf * L[j]) % r
            for k in range(self.ni):  # public-input rows nc + k: 1 * w[k] in A (reduction.rs:111-113)
                At[k] = (At[k] + L[self.nc + k]) % r
            for j, row in enumerate(b_rows):
                for cf, v in row:
                    Bt[v] = (Bt[v] + cf * L[j]) % r
            for j, row in enumerate(c_rows):
                for cf, v in row:
                    Ct[v] = (Ct[v] + cf * L[j]) % r
            dinv, ginv = pow(delta, r - 2, r), pow(gamma, r - 2, r)
            comb = [(beta * a + alpha * b + c) % r for a, b, c in zip(At, Bt, Ct)]
            l_sc = [x * dinv % r for x in comb[self.ni:]]
            ic_sc = [x * ginv % r for x in comb[:self.ni]]
            # h_query[i] = l_{2i+1}(tau) / delta over the 2n-domain (odd powers of w_2n)
            z2n = (pow(tau, 2 * n, r) - 1) % r
            odd, cur, w2sq = [], w_2n, w_2n * w_2n % r
            for _ in range(n):
                odd.append(cur)
                cur = cur * w2sq % r
            inv = _batch_inv([(2 * n * (tau - x)) % r for x in odd], r)
            h_sc = [z2n * x % r * iv % r * dinv % r for x, iv in zip(odd, inv)]
            if keep_trapdoor:
                self.At, self.Bt, self.Ct, self.h_sc = At, Bt, Ct, h_sc
        else:
            At = [rng.randrange(r) for _ in range(m)]
            Bt = [rng.randrange(r) for _ in range(m)]
            l_sc = [rng.randrange(r) for _ in range(m - self.ni)]
            self.c_rows = c_rows
            h_sc = [rng.randrange(r) for _ in range(n)]
            ic_sc = [rng.randrange(r) for _ in range(self.ni)]
        g1 = _fq_pts(list(cd.g1), 2, q, self.nq)[0]
        g2 = _fq_pts([cd.g2[0][0], cd.g2[0][1], cd.g2[1][0], cd.g2[1][1]], 4, q, self.nq)[0]
        fb = ctx.fixed_base_mul
        c = self.cid
        fr = self.fr
        a_fr, b_fr = fr(At), fr(Bt)
        small = fb(c, B.CS_G1, g1, fr([alpha, beta, delta] + ic_sc))
        small2 = fb(c, B.CS_G2, g2, fr([beta, gamma, delta]))
        self.points = dict(
            alpha_g1=small[0:1], beta_g1=small[1:2], delta_g1=small[2:3],
            beta_g2=small2[0:1], delta_g2=small2[2:3],
            a_query=fb(c, B.CS_G1, g1, a_fr), b_g1_query=fb(c, B.CS_G1, g1, b_fr),
            b_g2_query=fb(c, B.CS_G2, g2, b_fr),
            l_query=fb(c, B.CS_G1, g1, fr(l_sc)) if l_sc else np.zeros((0, 2 * self.nq), dtype=np.uint64),
            h_query=fb(c, B.CS_G1, g1, fr(h_sc)))
        self.gamma_g2 = small2[1:2]
        self.ic = small[3:3 + self.ni]

        def csr(rows):
            rp = np.zeros(len(rows) + 1, dtype=np.uint32)
            cols, cfs = [], []
            for i, row in enumerate(rows):
                for cf, v in row:
                    cols.append(v)
                    cfs.append(cf)
                rp[i + 1] = len(cols)
            return rp, np.array(cols, dtype=np.uint32), (fr(cfs) if cfs else np.zeros((0, 4), dtype=np.uint64))

        self.matrices = dict(num_constraints=self.nc, num_instance_variables=self.ni,
                             num_witness_variables=m - self.ni, a=csr(a_rows), b=csr(b_rows), c=csr(c_rows))
        self.public_inputs = fr(self.witness[:self.ni])
        self.private_witness = fr(self.witness[self.ni:])

    def fr(self, vals):
        """Scalars of this key's curve -> Montgomery limb array [len, 4]."""
        return _fr(vals, self.r)

    def make_key(self, window_bits=0):
        return B.Groth16Key(self.ctx, self.cid, self.matrices, self.points, window_bits)

    def vk_ints(self):
        """Verification key as oracle-style python tuples (for the pairing check in tests)."""
        def p1(a):
            v = B.from_mont_ints(B.limbs_to_ints(np.asarray(a).reshape(-1, self.nq)), self.q, self.nq)
            return None if not any(v) else (v[0], v[1])

        def p2(a):
            v = B.from_mont_ints(B.limbs_to_ints(np.asarray(a).reshape(-1, self.nq)), self.q, self.nq)
            return ((v[0], v[1]), (v[2], v[3]))

        return dict(alpha_g1=p1(self.points["alpha_g1"]), beta_g2=p2(self.points["beta_g2"]),
                    gamma_g2=p2(self.gamma_g2), delta_g2=p2(self.points["delta_g2"]),
                    ic=[p1(x) for x in self.ic])
