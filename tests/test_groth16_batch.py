"""Batched plain Groth16 (cs_groth16_prove_plain_batch): K witnesses of one circuit in one call.

Proof j of a batch must equal, byte for byte, cs_groth16_prove_plain on witness j with (r_j, s_j): the batch shares one
sort and one accumulation per MSM over K k B buckets (bucket (p k + g) B + d of proof p), runs the witness map over K
interleaved columns and does the single-point work on the device (k_point_*), so any mixing of proofs' buckets,
columns or terms shows as a differing proof.  Batches are of plain proofs only: the library has no Rep3 or Shamir batch.

CPU (emulation build): both curves at 2^6-2^8 with K in {1, 3, 17}, including an all-zero witness, two identical
witnesses in one batch and a public input of 0; a key with three public inputs and one with no witness; sub-batches
forced by the table budget; bad arguments; the prove CLI with three witness files.
GPU: K = 8 at 2^16 on both curves, identical to sequential proofs and accepted by the pairing check; a 2^20 batch large
enough to be split by the bucket limit; the prove CLI.
"""
import random

import numpy as np
import pytest

from co_snarks_b200 import binding as B
from helpers import Conv
from oracle import pairing_bls12_381, pairing_bn254
from workloads.synth_groth16 import SynthGroth16

ERR_ARG = -1  # CS_ERR_ARG
VERIFY = {"bn254": pairing_bn254.groth16_verify, "bls12_381": pairing_bls12_381.groth16_verify}


def batch_inputs(syn, K, seed):
    """K public-input and witness vectors for syn's key: the key's own witness first (its proof verifies), then an
    all-zero witness, a repeat of the first, a public input of 0, and random ones."""
    rng = random.Random(seed)
    r = syn.r
    nw = syn.private_witness.shape[0]
    pubs, wits = [], []
    for j in range(K):
        if j == 0 or j == 2:
            pub, wit = syn.witness[:syn.ni], syn.witness[syn.ni:]
        elif j == 1:
            pub, wit = [1] + [0] * (syn.ni - 1), [0] * nw
        elif j == 3:
            pub, wit = [1] + [0] * (syn.ni - 1), [rng.randrange(r) for _ in range(nw)]
        else:
            pub, wit = [1] + [rng.randrange(r) for _ in range(syn.ni - 1)], [rng.randrange(r) for _ in range(nw)]
        pubs.append(syn.fr(pub))
        wits.append(syn.fr(wit) if nw else np.zeros((0, 4), dtype=np.uint64))
    rs = [syn.fr([rng.randrange(r)]) for _ in range(K)]
    ss = [syn.fr([rng.randrange(r)]) for _ in range(K)]
    if K > 2:
        rs[2], ss[2] = rs[0], ss[0]  # a repeat of proof 0, blinders included: the two proofs must come out equal
    return np.stack(pubs), np.stack(wits), np.concatenate(rs), np.concatenate(ss)


def sequential(pk, pubs, wits, rs, ss):
    out = [pk.prove_plain(pubs[j], wits[j], rs[j:j + 1], ss[j:j + 1]) for j in range(len(pubs))]
    return tuple(np.stack([o[i] for o in out]) for i in range(3))


def check_batch(syn, pk, K, seed, verify=True):
    pubs, wits, rs, ss = batch_inputs(syn, K, seed)
    got = pk.prove_plain_batch(pubs, wits, rs, ss)
    exp = sequential(pk, pubs, wits, rs, ss)
    for g, e, name in zip(got, exp, "ABC"):
        assert g.shape == e.shape
        for j in range(K):
            assert np.array_equal(g[j], e[j]), "proof %d of %d: %s differs from the sequential proof" % (j, K, name)
    if K > 2:
        assert all(np.array_equal(got[i][0], got[i][2]) for i in range(3))
    if verify:
        cv = Conv(syn.curve)
        proof = (cv.pt1(got[0][0]), cv.pt2(got[1][0]), cv.pt1(got[2][0]))
        assert VERIFY[syn.curve](syn.vk_ints(), syn.witness[1:syn.ni], proof)
    return got


@pytest.mark.parametrize("curve,log_m", [("bn254", 6), ("bn254", 8), ("bls12_381", 6), ("bls12_381", 7)])
@pytest.mark.parametrize("K", [1, 3, 17])
def test_emu_batch_equals_sequential(emu_ctx, curve, log_m, K):
    syn = SynthGroth16(emu_ctx, log_m, curve=curve)
    pk = syn.make_key()
    try:
        check_batch(syn, pk, K, seed=K * 31 + log_m)
    finally:
        pk.free()


def test_emu_batch_several_public_inputs_and_no_witness(emu_ctx):
    """ni = 3 (two public terms per proof), and a key with no private witness (no witness MSMs: only H)"""
    r = Conv("bn254").r
    # x * y = z, z * 1 = w with x, y public; z, w private
    x, y = 12345, 678
    r1cs = ([[(1, 1)], [(1, 3)]], [[(1, 2)], [(1, 0)]], [[(1, 3)], [(1, 4)]], [1, x, y, x * y % r, x * y % r], 3)
    syn = SynthGroth16(emu_ctx, 0, r1cs=r1cs)
    pk = syn.make_key()
    try:
        check_batch(syn, pk, 5, seed=4)
    finally:
        pk.free()
    syn = SynthGroth16(emu_ctx, 0, r1cs=([[(1, 1)]], [[(1, 0)]], [[(1, 1)]], [1, 12345], 2))
    pk = syn.make_key()
    try:
        check_batch(syn, pk, 4, seed=5)
    finally:
        pk.free()


def test_emu_batch_split_by_budget(emu_ctx):
    """A budget too small for two proofs' scratch runs the batch one proof at a time: the same proofs, more launches."""
    syn = SynthGroth16(emu_ctx, 6)
    pk = syn.make_key()
    pubs, wits, rs, ss = batch_inputs(syn, 5, seed=8)
    try:
        l0 = emu_ctx.launch_count()
        whole = pk.prove_plain_batch(pubs, wits, rs, ss)
        l1 = emu_ctx.launch_count()
        emu_ctx.set_table_budget(1)
        split = pk.prove_plain_batch(pubs, wits, rs, ss)
        l2 = emu_ctx.launch_count()
    finally:
        emu_ctx.set_table_budget(0)
        pk.free()
    for a, b in zip(whole, split):
        assert np.array_equal(a, b)
    assert l2 - l1 > 3 * (l1 - l0), "the batch was not split (%d launches whole, %d split)" % (l1 - l0, l2 - l1)


def test_emu_batch_bad_arguments(emu_ctx):
    syn = SynthGroth16(emu_ctx, 5)
    pk = syn.make_key()
    lib = emu_ctx.lib
    pubs, wits, rs, ss = batch_inputs(syn, 2, seed=1)
    a = np.zeros((2, 8), dtype=np.uint64)
    b = np.zeros((2, 16), dtype=np.uint64)
    c = np.zeros((2, 8), dtype=np.uint64)
    P = B._ptr
    ni, nw = pubs.shape[1], wits.shape[1]
    try:
        def call(K=2, pub=pubs, n_pub=ni, wit=wits, d_wit=None, n_wit=nw, r=rs, s=ss, oa=a, ob=b, oc=c, ctx=None, key=None):
            return lib.cs_groth16_prove_plain_batch(ctx or emu_ctx.h, key or pk.h, K, P(pub), n_pub, P(wit), d_wit, n_wit,
                                                    P(r), P(s), P(oa), P(ob), P(oc))
        assert call() == 0
        assert call(K=0) == ERR_ARG
        assert call(n_wit=nw - 1) == ERR_ARG
        assert call(n_wit=nw + 1) == ERR_ARG
        assert call(n_pub=ni + 1) == ERR_ARG
        assert call(wit=None) == ERR_ARG
        assert call(d_wit=1) == ERR_ARG  # both a host and a device witness
        assert call(pub=None) == ERR_ARG
        assert call(r=None) == ERR_ARG
        assert call(oc=None) == ERR_ARG
        assert lib.cs_groth16_prove_plain_batch(None, pk.h, 2, P(pubs), ni, P(wits), None, nw, P(rs), P(ss), P(a), P(b),
                                                P(c)) == ERR_ARG
        assert lib.cs_groth16_prove_plain_batch(emu_ctx.h, None, 2, P(pubs), ni, P(wits), None, nw, P(rs), P(ss), P(a),
                                                P(b), P(c)) == ERR_ARG
        with pytest.raises(B.CsError):
            pk.prove_plain_batch(pubs[:0], wits[:0], rs[:0], ss[:0])
    finally:
        pk.free()


# ----------------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def gpu_ctx():
    ctx = B.Context(0)
    yield ctx
    ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("curve", ["bn254", "bls12_381"])
def test_gpu_batch_2p16(gpu_ctx, curve):
    syn = SynthGroth16(gpu_ctx, 16, curve=curve)
    pk = syn.make_key()
    try:
        pubs, wits, rs, ss = batch_inputs(syn, 8, seed=16)
        # the key's own witness with 8 different blinders: every proof must pass the pairing check
        pubs[:] = pubs[0]
        wits[:] = wits[0]
        got = pk.prove_plain_batch(pubs, wits, rs, ss)
        exp = sequential(pk, pubs, wits, rs, ss)
        for g, e in zip(got, exp):
            assert np.array_equal(g, e)
        cv = Conv(curve)
        for j in range(8):
            proof = (cv.pt1(got[0][j]), cv.pt2(got[1][j]), cv.pt1(got[2][j]))
            assert VERIFY[curve](syn.vk_ints(), syn.witness[1:syn.ni], proof)
        check_batch(syn, pk, 8, seed=17)  # the mixed batch (zero witness, repeats, public input 0)
    finally:
        pk.free()


@pytest.mark.gpu
def test_gpu_batch_2p20_split(gpu_ctx):
    """At 2^20 the witness MSMs take 2^15 buckets per proof: 40 proofs exceed the 2^20 bucket slots of one sort and
    run as sub-batches."""
    syn = SynthGroth16(gpu_ctx, 20)
    pk = syn.make_key()
    try:
        K = 40
        pubs, wits, rs, ss = batch_inputs(syn, K, seed=20)
        l0 = gpu_ctx.launch_count()
        got = pk.prove_plain_batch(pubs, wits, rs, ss)
        l1 = gpu_ctx.launch_count()
        got1 = pk.prove_plain_batch(pubs[:1], wits[:1], rs[:1], ss[:1])
        l2 = gpu_ctx.launch_count()
        assert l1 - l0 > l2 - l1, "the batch was not split"
        for g, g1 in zip(got, got1):
            assert np.array_equal(g[0], g1[0])
        exp = sequential(pk, pubs, wits, rs, ss)
        for g, e in zip(got, exp):
            assert np.array_equal(g, e)
    finally:
        pk.free()


# ----------------------------------------------------------------------------------------------------------- CLI
def run_cli(tmp_path, lib=None):
    """python -m co_snarks_b200.prove with three .wtns files: three proofs that the pairing check accepts"""
    import json
    import os
    import shutil

    from co_snarks_b200 import prove
    from helpers import golden_groth16, ih, reference_file
    from oracle import groth16 as OG
    base = "test_vectors/Groth16/bn254/poseidon/"
    zkey = reference_file(base + "circuit.zkey", tmp_path)
    w0 = reference_file(base + "witness.wtns", tmp_path)
    wtns = [w0] + [shutil.copy(w0, os.path.join(str(tmp_path), "w%d.wtns" % i)) for i in (1, 2)]
    out, pub = os.path.join(str(tmp_path), "proof.json"), os.path.join(str(tmp_path), "public.json")
    prove.main(["--zkey", zkey, "--wtns"] + wtns + ["--out", out, "--public-out", pub] + (["--lib", lib] if lib else []))
    z, _, _, g = golden_groth16("poseidon")
    vk = OG.vk_from_zkey(z)
    seen = set()
    for i in range(3):
        p = json.load(open(os.path.join(str(tmp_path), "proof_%d.json" % i)))
        public = [int(x) for x in json.load(open(os.path.join(str(tmp_path), "public_%d.json" % i)))]
        assert public == [ih(x) for x in g["public"]]
        a = (int(p["pi_a"][0]), int(p["pi_a"][1]))
        b = ((int(p["pi_b"][0][0]), int(p["pi_b"][0][1])), (int(p["pi_b"][1][0]), int(p["pi_b"][1][1])))
        c = (int(p["pi_c"][0]), int(p["pi_c"][1]))
        assert pairing_bn254.groth16_verify(vk, public, (a, b, c))
        seen.add(json.dumps(p))
    assert len(seen) == 3  # fresh (r, s) per proof
    assert not os.path.exists(out)


def test_emu_prove_cli_several_witnesses(tmp_path):
    import os
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
    import build_emu
    run_cli(tmp_path, lib=build_emu.build())


@pytest.mark.gpu
def test_gpu_prove_cli_several_witnesses(tmp_path):
    run_cli(tmp_path)
