"""Groth16 proofs checked exactly against the proof the known trapdoor implies, on BN254 and BLS12-381, at the sizes
production runs.

A key that workloads/synth_groth16.py builds from known (tau, alpha, beta, gamma, delta) has per-variable scalars
u_i(tau), v_i(tau), w_i(tau) (`At`, `Bt`, `Ct`).  For the full assignment z let U = sum z_i u_i(tau), V = sum z_i v_i(tau),
W = sum z_i w_i(tau).  For fixed (r, s) the proof is then unique:

    a = alpha + U + r delta,   b = beta + V + s delta,
    c = (sum_{i >= ni} z_i (beta u_i + alpha v_i + w_i) + U V - W) / delta + s a + r b - r s delta,
    proof = (a G1, b G2, c G1).

This holds for the circom reduction: h_query_i = L^{2n}_{2i+1}(tau) / delta, the circom h holds P = U V - W at the odd
2n-th roots of unity and P vanishes at the even ones, so sum_i h_i h_query_i = P(tau) / delta exactly.  The same identity
checks the witness map at any size: sum_i h_i h_sc_i must equal (U V - W) / delta, and since the device never sees tau,
a wrong h passes with probability about 1/r.  The reference below uses python integers and three scalar
multiplications in oracle.ec; it never calls the library.  It is pinned on the CPU against oracle/groth16.py and on the
GPU against oracle/c.

GPU keys are built in class-scoped fixtures and freed when their class is done: a 2^20 BLS12-381 key holds about 10 GB
of window tables, which is also why the Rep3 check, three keys at once, runs at 2^18.
"""
import random
import threading

import numpy as np
import pytest

from co_snarks_b200 import binding as B
from helpers import Conv
from kernel_checks import groth16_verifier
from oracle import groth16 as OG
from oracle.ec import g1 as og1, g2 as og2
from oracle.fields import CURVES
from workloads.synth_groth16 import SynthGroth16

CURVE_NAMES = ["bn254", "bls12_381"]


# ---------------------------------------------------------------------------------------------------- the reference
def trapdoor_scalars(syn, w):
    """-> (U, V, c without its (r, s) terms, (U V - W) / delta) for the full assignment w."""
    td, r = syn.trapdoor, syn.r
    alpha, beta, delta = td["alpha"], td["beta"], td["delta"]
    U = sum(x * y for x, y in zip(w, syn.At)) % r
    V = sum(x * y for x, y in zip(w, syn.Bt)) % r
    W = sum(x * y for x, y in zip(w, syn.Ct)) % r
    ni = syn.ni
    priv = (beta * sum(x * y for x, y in zip(w[ni:], syn.At[ni:])) + alpha * sum(x * y for x, y in zip(w[ni:], syn.Bt[ni:]))
            + sum(x * y for x, y in zip(w[ni:], syn.Ct[ni:]))) % r
    dinv = pow(delta, r - 2, r)
    return U, V, (priv + U * V - W) * dinv % r, (U * V - W) * dinv % r


def trapdoor_proof(syn, r_, s_):
    """The unique proof (A, B, C) for (r, s) and syn.witness, as oracle affine tuples."""
    td, r = syn.trapdoor, syn.r
    cd = CURVES[syn.curve]
    U, V, c0, _ = trapdoor_scalars(syn, syn.witness)
    a = (td["alpha"] + U + r_ * td["delta"]) % r
    b = (td["beta"] + V + s_ * td["delta"]) % r
    c = (c0 + s_ * a + r_ * b - r_ * s_ * td["delta"]) % r
    return og1(cd).mul(cd.g1, a), og2(cd).mul(cd.g2, b), og1(cd).mul(cd.g1, c)


def check_h_identity(syn, h):
    """sum_i h_i h_sc_i == (U V - W) / delta for the device's witness map output h (natural order)."""
    assert len(h) == syn.n == len(syn.h_sc)
    got = sum(x * y for x, y in zip(h, syn.h_sc)) % syn.r
    assert got == trapdoor_scalars(syn, syn.witness)[3], "witness map h fails the trapdoor identity"


def device_proof(syn, pk, r_, s_):
    cv = Conv(syn.curve)
    A, Bp, Cp = pk.prove_plain(syn.public_inputs, syn.private_witness, syn.fr([r_]), syn.fr([s_]))
    return cv.pt1(A), cv.pt2(Bp), cv.pt1(Cp)


def oracle_key(syn):
    """The synthetic key as the zkey-like dict and matrices oracle/groth16.py takes."""
    cv = Conv(syn.curve)
    p = syn.points
    g1s = lambda a: [cv.pt1(x) for x in np.asarray(a).reshape(-1, 2 * cv.nq)]
    g2s = lambda a: [cv.pt2(x) for x in np.asarray(a).reshape(-1, 4 * cv.nq)]
    z = dict(curve=CURVES[syn.curve], r=syn.r, q=syn.q)
    for k in ("alpha_g1", "beta_g1", "delta_g1"):
        z[k] = g1s(p[k])[0]
    for k in ("beta_g2", "delta_g2"):
        z[k] = g2s(p[k])[0]
    for k in ("a_query", "b_g1_query", "l_query", "h_query"):
        z[k] = g1s(p[k])
    z["b_g2_query"] = g2s(p["b_g2_query"])
    m = dict(num_constraints=syn.nc, num_instance_variables=syn.ni, num_witness_variables=syn.m - syn.ni,
             a=syn.a_rows, b=syn.b_rows)
    return z, m


def oracle_c_desc(syn):
    from oracle.c import run as OC
    return OC.key_desc(syn.matrices, syn.points, curve=syn.cid)


# ---------------------------------------------------------------------------------------------------- circuits
def realistic_r1cs(curve, n_values, run, n_pub=64, seed=31):
    """An explicit R1CS shaped like real circuits rather than the random chain:
    - n_pub public inputs, each squared by one constraint;
    - n_values 64-bit values, each bit-decomposed: b * (b - 1) = 0 per bit (rows with an empty C) and one packing row
      (sum 2^t b_t) * 1 = x, so most witness scalars are 0 or 1;
    - a run of `run` equal witness values y_{k+1} = y_k * 1 (one bucket of every window takes them all);
    - one witness variable that occurs in no constraint (its A, B and L bases are the point at infinity).
    -> (a_rows, b_rows, c_rows, witness, num_instance_variables)."""
    r = CURVES[curve].r
    rng = random.Random(seed)
    small = min(c.r for c in CURVES.values())  # the same witness on both curves
    w = [1] + [rng.randrange(small) for _ in range(n_pub)]
    a, b, c = [], [], []

    def var(v):
        w.append(v % r)
        return len(w) - 1

    var(rng.randrange(small))  # the unused variable
    for k in range(1, n_pub + 1):
        sq = var(w[k] * w[k])
        a.append([(1, k)])
        b.append([(1, k)])
        c.append([(1, sq)])
    for _ in range(n_values):
        x = rng.getrandbits(64)
        xv = var(x)
        bits = [var((x >> t) & 1) for t in range(64)]
        for bv in bits:
            a.append([(1, bv)])
            b.append([(1, bv), (r - 1, 0)])
            c.append([])
        a.append([(1 << t, bv) for t, bv in enumerate(bits)])
        b.append([(1, 0)])
        c.append([(1, xv)])
    y = var(w[1] * w[2])
    a.append([(1, 1)])
    b.append([(1, 2)])
    c.append([(1, y)])
    for _ in range(run - 1):
        y2 = var(w[y])
        a.append([(1, y)])
        b.append([(1, 0)])
        c.append([(1, y2)])
        y = y2
    return a, b, c, w, n_pub + 1


def satisfied(syn):
    """Every row of the system holds for syn.witness (so the trapdoor formula applies)."""
    w, r = syn.witness, syn.r
    rows_c = syn.matrices["c"]
    rp, col = rows_c[0], rows_c[1]
    cvals = Conv(syn.curve).fr_back(rows_c[2]) if len(col) else []
    for j, (ra, rb) in enumerate(zip(syn.a_rows, syn.b_rows)):
        av = sum(cf * w[v] for cf, v in ra) % r
        bv = sum(cf * w[v] for cf, v in rb) % r
        cc = sum(cvals[k] * w[col[k]] for k in range(rp[j], rp[j + 1])) % r
        if av * bv % r != cc:
            return False
    return True


# ---------------------------------------------------------------------------------------------------- CPU: pin the reference
@pytest.mark.parametrize("curve", CURVE_NAMES)
def test_trapdoor_reference_equals_oracle_emu(emu_ctx, curve):
    """At 2^6 the trapdoor proof equals oracle/groth16.py's prove_plain for the same key and (r, s), passes the curve's
    pairing check, and equals the emulated device proof; the device h passes the H identity."""
    syn = SynthGroth16(emu_ctx, 6, curve=curve, keep_trapdoor=True)
    assert satisfied(syn)
    z, m = oracle_key(syn)
    vk = syn.vk_ints()
    pk = syn.make_key()
    rng = random.Random(41)
    for r_, s_ in ((0, 0), (rng.randrange(syn.r), rng.randrange(syn.r))):
        exp = trapdoor_proof(syn, r_, s_)
        assert OG.prove_plain(z, m, syn.witness, r_, s_) == exp
        assert groth16_verifier(curve)(vk, syn.witness[1:2], exp)
        assert device_proof(syn, pk, r_, s_) == exp
    check_h_identity(syn, Conv(curve).fr_back(pk.witness_map(syn.public_inputs, syn.private_witness)))
    pk.free()


@pytest.mark.parametrize("curve", CURVE_NAMES)
def test_trapdoor_reference_rejects_unsatisfied_witness_emu(emu_ctx, curve):
    """With one witness value changed so that its constraint fails, the trapdoor formula no longer gives the oracle's
    proof (the circom reduction interpolates A z .* B z, not C z), and the device h fails the H identity."""
    syn = SynthGroth16(emu_ctx, 6, curve=curve, keep_trapdoor=True)
    z, m = oracle_key(syn)
    k = syn.m - 1  # defined by the last constraint and used by none
    syn.witness = list(syn.witness)
    syn.witness[k] = (syn.witness[k] + 1) % syn.r
    assert not satisfied(syn)
    r_, s_ = 5, 7
    assert OG.prove_plain(z, m, syn.witness, r_, s_) != trapdoor_proof(syn, r_, s_)
    syn.private_witness = syn.fr(syn.witness[syn.ni:])
    pk = syn.make_key()
    h = Conv(curve).fr_back(pk.witness_map(syn.public_inputs, syn.private_witness))
    with pytest.raises(AssertionError):
        check_h_identity(syn, h)
    pk.free()


def test_synth_any_constraint_count_emu(emu_ctx):
    """The seeded chain at a constraint count that is not 2^k - 2: 2^5 + 1 rows give a 2^6 domain, half of it padding.
    The proof equals the trapdoor proof, and h equals oracle/c's BLS12-381 witness map and passes the H identity."""
    from oracle.c import run as OC
    syn = SynthGroth16(emu_ctx, 0, curve="bls12_381", num_constraints=31, keep_trapdoor=True)
    assert (syn.nc, syn.m, syn.n) == (31, 33, 64) and satisfied(syn)
    pk = syn.make_key()
    assert pk.domain_size() == 64
    assert device_proof(syn, pk, 3, 4) == trapdoor_proof(syn, 3, 4)
    h = pk.witness_map(syn.public_inputs, syn.private_witness)
    desc, keep = oracle_c_desc(syn)
    assert np.array_equal(h, OC.witness_map(desc, 0, 0, syn.public_inputs, syn.private_witness))
    check_h_identity(syn, Conv("bls12_381").fr_back(h))
    pk.free()


@pytest.mark.parametrize("curve", CURVE_NAMES)
def test_realistic_circuit_small_emu(emu_ctx, curve):
    """The realistic circuit's shapes at a small size (3 decomposed values, a run of 40, 64 public inputs): the oracle,
    the trapdoor reference and the emulated device agree."""
    syn = SynthGroth16(emu_ctx, 0, r1cs=realistic_r1cs(curve, 3, 40), curve=curve, keep_trapdoor=True)
    assert satisfied(syn) and syn.ni == 65 and syn.n == 512
    z, m = oracle_key(syn)
    pk = syn.make_key()
    exp = trapdoor_proof(syn, 11, 13)
    assert OG.prove_plain(z, m, syn.witness, 11, 13) == exp
    assert device_proof(syn, pk, 11, 13) == exp
    pk.free()


# ---------------------------------------------------------------------------------------------------- GPU
def _free_after(syn, pk):
    pk.free()
    syn.points = None


@pytest.mark.gpu
def test_trapdoor_reference_equals_oracle_c_bn254_gpu(gpu_ctx):
    """BN254 at 2^12: the trapdoor proof equals oracle/c's prove_plain byte for byte, and the device proof equals both."""
    from oracle.c import run as OC
    cv = Conv("bn254")
    syn = SynthGroth16(gpu_ctx, 12, keep_trapdoor=True)
    desc, keep = oracle_c_desc(syn)
    pk = syn.make_key()
    for r_, s_ in ((0, 0), (123456789, 987654321)):
        a, b, c = OC.prove_plain(desc, syn.public_inputs, syn.private_witness, syn.fr([r_]), syn.fr([s_]))
        exp = trapdoor_proof(syn, r_, s_)
        assert (cv.pt1(a), cv.pt2(b), cv.pt1(c)) == exp
        assert device_proof(syn, pk, r_, s_) == exp
    _free_after(syn, pk)
    del keep


@pytest.fixture(scope="class")
def production_key(gpu_ctx):
    syn = SynthGroth16(gpu_ctx, 20, curve="bls12_381", keep_trapdoor=True)
    pk = syn.make_key()
    yield syn, pk
    _free_after(syn, pk)


@pytest.fixture(scope="class")
def domain_edge_key(gpu_ctx):
    syn = SynthGroth16(gpu_ctx, 0, curve="bls12_381", num_constraints=(1 << 20) - 1, keep_trapdoor=True)
    assert syn.n == 1 << 21 and syn.nc + syn.ni == (1 << 20) + 1
    pk = syn.make_key()
    yield syn, pk
    _free_after(syn, pk)


@pytest.mark.gpu
class TestBls12381ProductionSize:
    """BLS12-381, the bench's chain R1CS with a full 2^20 domain."""

    @pytest.fixture
    def key(self, production_key):
        return production_key

    @pytest.mark.parametrize("rs", [(0, 0), (0x1d2c3b4a5968778695a4b3c2d1e0f, 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfefffffffeffffffff)])
    def test_proof(self, key, rs):
        syn, pk = key
        assert device_proof(syn, pk, *rs) == trapdoor_proof(syn, *rs)

    def test_h_identity(self, key):
        syn, pk = key
        check_h_identity(syn, Conv(syn.curve).fr_back(pk.witness_map(syn.public_inputs, syn.private_witness)))


@pytest.mark.gpu
class TestBls12381DomainEdge:
    """BLS12-381 with 2^20 + 1 rows: a 2^21 domain that is half padding, so the witness map runs three NTT passes with
    the coset table applied in the last one."""

    @pytest.fixture
    def key(self, domain_edge_key):
        return domain_edge_key

    def test_proof(self, key):
        syn, pk = key
        assert device_proof(syn, pk, 31337, 271828) == trapdoor_proof(syn, 31337, 271828)

    def test_witness_map_against_oracle_c(self, key):
        """pk.witness_map element by element against oracle/c's BLS12-381 witness map, and the H identity."""
        from oracle.c import run as OC
        syn, pk = key
        h = pk.witness_map(syn.public_inputs, syn.private_witness)
        desc, keep = oracle_c_desc(syn)
        exp = OC.witness_map(desc, 0, 0, syn.public_inputs, syn.private_witness)
        if not np.array_equal(h, exp):
            bad = np.nonzero((h != exp).any(axis=1))[0]
            raise AssertionError("witness map: %d of %d elements differ, first at %s" % (bad.size, syn.n, bad[:4].tolist()))
        check_h_identity(syn, Conv(syn.curve).fr_back(h))
        del keep


def _realistic(ctx, curve):
    return SynthGroth16(ctx, 0, r1cs=realistic_r1cs(curve, 2000, (1 << 16) + 3), curve=curve, keep_trapdoor=True)


def _check_realistic_shape(syn):
    w = syn.witness[syn.ni:]
    assert syn.ni - 1 >= 64
    assert sum(1 for x in w if x in (0, 1)) >= 0.4 * len(w)
    assert syn.n // 2 < syn.nc + syn.ni < syn.n == 1 << 18  # about 2^18, not full
    assert (np.diff(syn.matrices["c"][0]) == 0).any()  # rows with an empty C
    run = best = 1
    for x, y in zip(w, w[1:]):
        run = run + 1 if x == y else 1
        best = max(best, run)
    assert best >= 1 << 16
    used = np.zeros(syn.m, dtype=bool)
    for k in ("a", "b", "c"):
        used[syn.matrices[k][1]] = True
    assert not used.all()  # a witness variable in no constraint


@pytest.mark.gpu
@pytest.mark.parametrize("curve", CURVE_NAMES)
def test_realistic_circuit_gpu(gpu_ctx, curve):
    """The realistic circuit at about 2^18 (bit decompositions, a run of 2^16 + 3 equal values, 64 public inputs, empty
    C rows, an unused variable, a 3/4-full domain): the proof equals the trapdoor proof and h passes the H identity;
    on BN254 the proof also equals oracle/c's byte for byte."""
    syn = _realistic(gpu_ctx, curve)
    _check_realistic_shape(syn)
    assert satisfied(syn)
    pk = syn.make_key()
    exp = trapdoor_proof(syn, 987654321, 123456789)
    assert device_proof(syn, pk, 987654321, 123456789) == exp
    check_h_identity(syn, Conv(curve).fr_back(pk.witness_map(syn.public_inputs, syn.private_witness)))
    if curve == "bn254":
        from oracle.c import run as OC
        cv = Conv(curve)
        desc, keep = oracle_c_desc(syn)
        a, b, c = OC.prove_plain(desc, syn.public_inputs, syn.private_witness, syn.fr([987654321]), syn.fr([123456789]))
        assert (cv.pt1(a), cv.pt2(b), cv.pt1(c)) == exp
        del keep
    _free_after(syn, pk)


@pytest.mark.gpu
def test_rep3_realistic_bls12_381_gpu(gpu_ctx):
    """Rep3 on BLS12-381 at 2^18 on the realistic circuit: three party threads on one GPU through rep3_prove.  All
    parties return the same proof, it equals the trapdoor proof for (sum r_i, sum s_i), the replicated r / s shares are
    consistent, and each net carries less than 2 KB (points only)."""
    syn = _realistic(gpu_ctx, "bls12_381")
    cv = Conv(syn.curve)
    r = syn.r
    ni = syn.ni
    ctxs = [B.Context(0) for _ in range(3)]
    pks = [B.Groth16Key(c, syn.cid, syn.matrices, syn.points) for c in ctxs]
    nets0 = [B.Net.peer(ctxs[i], i, 3) for i in range(3)]
    nets1 = [B.Net.peer(ctxs[i], i, 3) for i in range(3)]
    for i in range(3):
        nets0[i].connect_local(nets0)
        nets1[i].connect_local(nets1)
    lib = ctxs[0].lib
    seeds = [bytes([29 * (i + 1) + k for k in range(32)]) for i in range(3)]
    states = [B.Rep3StateC.from_seeds(lib, i, seeds[i], seeds[(i + 2) % 3]) for i in range(3)]
    wsh = OG.share_rep3(syn.witness[ni:], r, random.Random(43))
    shares = [syn.fr([x for ab in wsh[i] for x in ab]).reshape(-1, 8) for i in range(3)]
    out, errs = {}, []

    def party(i):
        try:
            A, Bp, Cp, rs = pks[i].rep3_prove(nets0[i], nets1[i], states[i], syn.public_inputs, shares[i], want_rs=True)
            out[i] = ((cv.pt1(A), cv.pt2(Bp), cv.pt1(Cp)), cv.fr_back(rs))
        except Exception as e:  # noqa: BLE001
            errs.append(e)
    th = [threading.Thread(target=party, args=(i,)) for i in range(3)]
    for t in th:
        t.start()
    for t in th:
        t.join(timeout=900)
    try:
        assert not errs, errs
        assert len(out) == 3
        proofs = [out[i][0] for i in range(3)]
        assert proofs[0] == proofs[1] == proofs[2], "parties disagree on the proof"
        rs = [out[i][1] for i in range(3)]
        for i in range(3):
            assert rs[i][1] == rs[(i + 2) % 3][0] and rs[i][3] == rs[(i + 2) % 3][2], "r / s shares are not replicated"
        r_tot, s_tot = sum(x[0] for x in rs) % r, sum(x[2] for x in rs) % r
        assert proofs[0] == trapdoor_proof(syn, r_tot, s_tot), "opened Rep3 proof != trapdoor proof for (sum r, sum s)"
        sent = [n.bytes_sent for n in nets0 + nets1]
        assert all(0 < s < 2048 for s in sent), sent
    finally:
        for pk in pks:
            pk.free()
        for n in nets0 + nets1:
            n.free()
        for s in states:
            s.free()
        for c in ctxs:
            c.close()
