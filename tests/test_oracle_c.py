"""CPU-only: the C restatement (oracle/c, the timed CPU baseline) against the Python oracle and the
golden vectors -- identical proofs for fixed (r, s) on the reference's Groth16 fixtures."""
import random

import numpy as np
import pytest

from helpers import Conv, golden_groth16, ih
from oracle import groth16 as OG
from oracle import ntt as ON
from oracle.c import run as OC
from oracle.ec import g1 as og1, g2 as og2
from oracle.fields import BN254, groth16_roots_of_unity
from oracle.formats import proof_to_json


def test_c_msm_matches_python_oracle():
    cv = Conv("bn254")
    rng = random.Random(1)
    for group, G, gen, to_arr, to_pt, n in ((0, og1(BN254), BN254.g1, cv.g1, cv.pt1, 200), (1, og2(BN254), BN254.g2, cv.g2, cv.pt2, 60)):
        pts = [G.mul(gen, rng.randrange(1, cv.r)) for _ in range(n)]
        pts[3] = None
        pts[5] = pts[4]
        sc = [rng.randrange(cv.r) for _ in range(n)]
        sc[0], sc[1], sc[4], sc[5] = 0, cv.r - 1, 9, 9
        out = OC.msm(to_arr(pts), cv.fr(sc), group)
        assert to_pt(out) == G.msm(pts, sc)


def _c_ntt_matches_python_oracle(curve, log_sizes, seed):
    cv = Conv(curve)
    rng = random.Random(seed)
    for lg in log_sizes:
        n = 1 << lg
        g, _ = groth16_roots_of_unity(cv.r, lg)
        for batch in (1, 2):
            v = [rng.randrange(cv.r) for _ in range(n * batch)]
            if n * batch >= 4:
                v[:4] = [0, 1, cv.r - 1, cv.r - 2]
            arr = cv.fr(v)
            OC.ifft_in_to_out(arr, lg, batch, cv.fr([g]), curve=cv.id)
            exp = [None] * (n * batch)
            for c in range(batch):
                exp[c::batch] = ON.ifft_in_to_out(v[c::batch], g, cv.r)
            assert cv.fr_back(arr) == exp, (curve, lg, batch)
            OC.fft_out_to_in(arr, lg, batch, cv.fr([g]), curve=cv.id)
            assert cv.fr_back(arr) == v, (curve, lg, batch)
            # the forward transform on its own input (a round trip cannot show an error both directions share)
            w = [rng.randrange(cv.r) for _ in range(n * batch)]
            arr = cv.fr(w)
            OC.fft_out_to_in(arr, lg, batch, cv.fr([g]), curve=cv.id)
            for c in range(batch):
                nat = ON.bit_reverse_perm(w[c::batch])
                assert cv.fr_back(arr[c::batch]) == [sum(x * pow(g, i * j, cv.r) for j, x in enumerate(nat)) % cv.r
                                                     for i in range(n)], (curve, lg, batch)


def test_c_ntt_matches_python_oracle():
    _c_ntt_matches_python_oracle("bn254", (1, 4, 9), 2)


def test_c_ntt_bls12_381_matches_python_oracle():
    """oracle/c's BLS12-381 Fr context (4 x 64-bit limbs, 255-bit r) against the Python oracle and the definition."""
    _c_ntt_matches_python_oracle("bls12_381", (1, 2, 5, 8), 3)


@pytest.mark.parametrize("name", ["multiplier2", "poseidon"])
def test_c_groth16_equals_golden_proof(name):
    cv = Conv("bn254")
    z, m, w, g = golden_groth16(name)
    ni = m["num_instance_variables"]
    mats = dict(num_constraints=m["num_constraints"], num_instance_variables=ni,
                num_witness_variables=m["num_witness_variables"], a=cv.csr(m["a"]), b=cv.csr(m["b"]))
    pts = dict(alpha_g1=cv.g1([z["alpha_g1"]]), beta_g1=cv.g1([z["beta_g1"]]), beta_g2=cv.g2([z["beta_g2"]]),
               delta_g1=cv.g1([z["delta_g1"]]), delta_g2=cv.g2([z["delta_g2"]]), a_query=cv.g1(z["a_query"]),
               b_g1_query=cv.g1(z["b_g1_query"]), b_g2_query=cv.g2(z["b_g2_query"]), l_query=cv.g1(z["l_query"]),
               h_query=cv.g1(z["h_query"]))
    desc, keep = OC.key_desc(mats, pts)
    pub, wit = cv.fr(w[:ni]), cv.fr(w[ni:])
    assert cv.fr_back(OC.witness_map(desc, 0, 0, pub, wit)) == [ih(x) for x in g["h"]]
    for pr in g["oracle_proofs"]:
        a, b, c = OC.prove_plain(desc, pub, wit, cv.fr([ih(pr["r"])]), cv.fr([ih(pr["s"])]))
        assert proof_to_json(cv.pt1(a), cv.pt2(b), cv.pt1(c)) == pr["json"]
    # Rep3 witness map shares
    rng = random.Random(5)
    wsh = OG.share_rep3(w[ni:], cv.r, rng)
    n = len(g["h"])
    m1 = [rng.randrange(cv.r) for _ in range(n)]
    m2 = [rng.randrange(cv.r) for _ in range(n)]
    for party in range(3):
        sh = cv.fr([x for ab in wsh[party] for x in ab])
        got = cv.fr_back(OC.witness_map(desc, 1, party, pub, sh, cv.fr(m1), cv.fr(m2)))
        assert got == OG.witness_map_rep3(party, m, w[:ni], wsh[party], m1, m2, cv.r, 28)


@pytest.mark.parametrize("name", ["multiplier2", "poseidon"])
def test_c_witness_map_bls12_381_equals_golden(name):
    """oracle_witness_map on a BLS12-381 key (key_desc curve 1): its Fr, two-adicity 32 and that field's roots and
    coset shift give the golden h of the reference's BLS12-381 fixture, plain and as Rep3 shares."""
    cv = Conv("bls12_381")
    z, m, w, g = golden_groth16(name, "bls12_381")
    ni = m["num_instance_variables"]
    mats = dict(num_constraints=m["num_constraints"], num_instance_variables=ni,
                num_witness_variables=m["num_witness_variables"], a=cv.csr(m["a"]), b=cv.csr(m["b"]))
    desc, keep = OC.key_desc(mats, {k: np.zeros((1, 24), dtype=np.uint64) for k in (
        "alpha_g1", "beta_g1", "beta_g2", "delta_g1", "delta_g2", "a_query", "b_g1_query", "b_g2_query", "l_query",
        "h_query")}, curve=cv.id)
    pub, wit = cv.fr(w[:ni]), cv.fr(w[ni:])
    assert cv.fr_back(OC.witness_map(desc, 0, 0, pub, wit)) == [ih(x) for x in g["h"]]
    rng = random.Random(6)
    wsh = OG.share_rep3(w[ni:], cv.r, rng)
    n = len(g["h"])
    m1 = [rng.randrange(cv.r) for _ in range(n)]
    m2 = [rng.randrange(cv.r) for _ in range(n)]
    for party in range(3):
        got = cv.fr_back(OC.witness_map(desc, 1, party, pub, cv.fr([x for ab in wsh[party] for x in ab]), cv.fr(m1), cv.fr(m2)))
        assert got == OG.witness_map_rep3(party, m, w[:ni], wsh[party], m1, m2, cv.r, 32)
    # a BLS12-381 key cannot go through the BN254-only prover
    with pytest.raises(AssertionError):
        OC.prove_plain(desc, pub, wit, cv.fr([1]), cv.fr([2]))


@pytest.mark.parametrize("name", ["multiplier2", "poseidon"])
def test_c_plonk_prover_matches_python_oracle_and_kats(name):
    """oracle/c/plonk.inc (the CPU baseline of the Plonk row) == oracle/plonk.py == the reference's known answers."""
    from helpers import golden_plonk, plonk_key_arrays, plonk_proof_from_device
    from oracle.formats import plonk_proof_to_json
    cv = Conv("bn254")
    z, w, g = golden_plonk(name)
    npub = z["n_public"]
    pts, evs = OC.plonk_prove(plonk_key_arrays(cv, z), cv.fr(w[:npub + 1]), cv.fr(w[npub + 1:]), cv.fr(list(range(11))))
    assert plonk_proof_to_json(plonk_proof_from_device(cv, pts, evs)) == g["oracle_proof_json"]
