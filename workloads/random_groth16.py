"""BN254 Groth16 keys of any size built vectorised (numpy and cs_fixed_base_mul), for checks and timings at sizes where
SynthGroth16's Python-integer setup would take many minutes and tens of GB of host memory; and the least table budget
that leaves a key a given number of table rows."""
import numpy as np

from co_snarks_b200 import binding as B
from oracle.fields import CURVES

ERR_LIMIT = -3


def _mont(vals, q):
    return B.ints_to_limbs(B.to_mont_ints(vals, q, 4), 4).reshape(-1)


def rand_fr_limbs(rng, n):
    """n elements below 2^252 < r (BN254), as 4 little-endian limbs; any value below r is a Montgomery form"""
    x = rng.integers(0, 1 << 63, size=(n, 4), dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, size=(n, 4), dtype=np.uint64)
    x[:, 3] &= np.uint64((1 << 60) - 1)
    return x


def random_key(ctx, lg, seed=24):
    """A BN254 Groth16 key with a 2^lg domain built vectorised: nc + ni = 2^lg rows of two random entries in A and B,
    random witness, query points k G for random k from cs_fixed_base_mul (a pool per group, rolled per query; some B
    bases at infinity).  The witness does not satisfy the R1CS: oracle/c computes the same function either way."""
    rng = np.random.default_rng(seed)
    ni = 4
    n = 1 << lg
    nc, nw = n - ni, n - ni
    m = ni + nw
    cd = CURVES["bn254"]
    gen1 = _mont([cd.g1[0], cd.g1[1]], cd.q)
    gen2 = _mont([cd.g2[0][0], cd.g2[0][1], cd.g2[1][0], cd.g2[1][1]], cd.q)

    def csr():
        rp = np.arange(0, 2 * nc + 1, 2, dtype=np.uint32)
        col = rng.integers(0, m, size=2 * nc, dtype=np.uint32)
        return rp, col, rand_fr_limbs(rng, 2 * nc)

    mats = dict(num_constraints=nc, num_instance_variables=ni, num_witness_variables=nw, a=csr(), b=csr())
    g1 = ctx.fixed_base_mul(B.CS_BN254, 0, gen1, rand_fr_limbs(rng, n), montgomery=False)
    g2 = ctx.fixed_base_mul(B.CS_BN254, 1, gen2, rand_fr_limbs(rng, m), montgomery=False)
    b1 = np.roll(g1, 3, axis=0)[:m].copy()
    inf = rng.integers(0, m, size=64)
    b1[inf] = 0
    g2[inf] = 0
    pts = dict(alpha_g1=g1[1:2], beta_g1=g1[2:3], beta_g2=g2[1:2], delta_g1=g1[3:4], delta_g2=g2[2:3],
               a_query=np.roll(g1, 1, axis=0)[:m].copy(), b_g1_query=b1, b_g2_query=g2,
               l_query=np.roll(g1, 2, axis=0)[:nw].copy(), h_query=g1)
    pub = rand_fr_limbs(rng, ni)
    wit = rand_fr_limbs(rng, nw)
    return mats, pts, pub, wit


def forced_key(ctx, make, rows):
    """The key make() builds with the largest table budget that leaves it at most `rows` table rows, i.e. with the
    smallest k of that row count.  A larger budget gives more rows and a smaller one fewer or CS_ERR_LIMIT, so the
    budgets that work form an interval below the one that gives more rows; on tiny keys, whose scratch grows with k
    faster than their tables shrink, it is empty.  Leaves the budget set to the one found."""
    pk = make()
    full_rows, full_bytes = pk.table_info()
    pk.free()
    lo, hi, good = 0, 4 * full_bytes + (64 << 20), None  # hi: more rows than wanted
    while hi - lo > max(1, hi >> 16):
        mid = (lo + hi) // 2
        ctx.set_table_budget(mid)
        try:
            pk = make()
        except B.CsError as e:
            assert "error %d" % ERR_LIMIT in str(e), e
            lo = mid
            continue
        r = pk.table_info()[0]
        pk.free()
        if r <= rows:
            lo = good = mid
        else:
            hi = mid
    assert good is not None, "no table budget leaves the key at most %d of %d rows" % (rows, full_rows)
    ctx.set_table_budget(good)
    return make()
