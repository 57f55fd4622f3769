"""GPU tests at BASELINE.json's full sizes (2^20), checked through size-independent properties:
  * MSM over bases k_i*G equals (sum s_i k_i)*G  -- one oracle scalar multiplication pins 2^20 terms;
  * NTT round trip and the convolution-free identity  NTT(a + b) = NTT(a) + NTT(b)  at 2^20;
  * a 2^20-constraint Groth16 proof from a known-toxic-waste key passes the BN254 pairing check."""
import random

import numpy as np
import pytest

from co_snarks_b200 import binding as B
import kernel_checks as K
from helpers import Conv
from oracle.ec import g1 as og1, g2 as og2
from oracle.fields import BN254, groth16_roots_of_unity
from oracle.pairing_bn254 import groth16_verify

pytestmark = pytest.mark.gpu


def _rand_fr_limbs(n, seed, r):
    """n uniform field elements as canonical limbs, vectorised (rejection-free: 253-bit draws < r)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    a = rng.integers(0, 2 ** 63, size=(n, 4), dtype=np.uint64) << np.uint64(1)
    a |= rng.integers(0, 2, size=(n, 4), dtype=np.uint64)
    a[:, 3] &= np.uint64((1 << 61) - 1)  # < 2^253 < r
    return a


def _sum_products(s_limbs, k_limbs, r):
    s = B.limbs_to_ints(s_limbs)
    k = B.limbs_to_ints(k_limbs)
    return sum(x * y for x, y in zip(s, k)) % r


@pytest.mark.parametrize("group,logn", [(0, 20), (1, 18)])
def test_msm_fullsize_known_dlog(gpu_ctx, group, logn):
    cv = Conv("bn254")
    n = 1 << logn
    k = _rand_fr_limbs(n, 100 + group, cv.r)
    s = _rand_fr_limbs(n, 200 + group, cv.r)
    G = og1(BN254) if group == 0 else og2(BN254)
    gen = BN254.g1 if group == 0 else BN254.g2
    gen_arr = (cv.g1 if group == 0 else cv.g2)([gen])[0]
    pts = gpu_ctx.fixed_base_mul(cv.id, group, gen_arr, k, montgomery=False)
    bases = gpu_ctx.bases_upload(cv.id, group, pts)
    out, inf = gpu_ctx.msm(bases, s, montgomery=False)
    exp = G.mul(gen, _sum_products(s, k, cv.r))
    assert (cv.pt1 if group == 0 else cv.pt2)(out) == exp
    # linearity on a second scalar vector: msm(s) + msm(t) == msm(s + t mod r) -- checked via dlogs too
    t = _rand_fr_limbs(n, 300 + group, cv.r)
    out2, _ = gpu_ctx.msm(bases, t, montgomery=False)
    exp2 = G.mul(gen, _sum_products(t, k, cv.r))
    assert (cv.pt1 if group == 0 else cv.pt2)(out2) == exp2
    bases.free()


def test_ntt_fullsize_roundtrip_and_linearity(gpu_ctx):
    cv = Conv("bn254")
    lg = 20
    n = 1 << lg
    g, _ = groth16_roots_of_unity(cv.r, lg)
    dom = gpu_ctx.domain(cv.id, lg, cv.fr([g]))
    a = _rand_fr_limbs(n, 1, cv.r)  # treated as Montgomery representations of some elements
    b = _rand_fr_limbs(n, 2, cv.r)
    lib = gpu_ctx.lib
    da, db = gpu_ctx.to_device(a), gpu_ctx.to_device(b)
    dsum = gpu_ctx.alloc(n * 32)
    gpu_ctx._check(lib.cs_vec_add(gpu_ctx.h, cv.id, da, db, dsum, n))
    for d in (da, db, dsum):
        dom.ifft_in_to_out(d, 1)
    dchk = gpu_ctx.alloc(n * 32)
    gpu_ctx._check(lib.cs_vec_add(gpu_ctx.h, cv.id, da, db, dchk, n))
    assert (gpu_ctx.d2h(dchk, (n, 4)) == gpu_ctx.d2h(dsum, (n, 4))).all(), "iNTT is not linear"
    dom.fft_out_to_in(da, 1)
    assert (gpu_ctx.d2h(da, (n, 4)) == a).all(), "NTT(iNTT(a)) != a at 2^20"
    # spot-check 4 outputs of the forward transform against the definition  X_i = sum_j x_j g^(ij)
    x = B.from_mont_ints(B.limbs_to_ints(b[:]), cv.r, 4)
    dom.fft_out_to_in(db, 1)  # db holds iNTT(b) in bit-reversed order -> back to b
    assert (gpu_ctx.d2h(db, (n, 4)) == b).all()
    dnat = gpu_ctx.to_device(b)
    gpu_ctx._check(lib.cs_bit_reverse(gpu_ctx.h, cv.id, dnat, lg, 1))
    dom.fft_out_to_in(dnat, 1)  # forward NTT of b (natural in after the explicit bit reversal)
    got = gpu_ctx.d2h(dnat, (n, 4))
    for i in (0, 1, 12345, n - 1):
        gi = pow(g, i, cv.r)
        acc, p = 0, 1
        for xj in x:
            acc += xj * p
            p = p * gi % cv.r
        assert cv.fr_back(got[i:i + 1]) == [acc % cv.r]
    for d in (da, db, dsum, dchk, dnat):
        gpu_ctx.free(d)
    dom.free()


@pytest.fixture(scope="module")
def syn20(gpu_ctx):
    """BASELINE configs[1]/[2]: the synthetic 2^20-constraint R1CS with a valid (known toxic waste) key."""
    from workloads.synth_groth16 import SynthGroth16
    return SynthGroth16(gpu_ctx, 20)


def test_groth16_2p20_proof_bytes_equal_oracle_c(gpu_ctx, syn20):
    """Bit-exact at BASELINE size: the GPU proof at 2^20 constraints equals the proof of the CPU restatement
    (oracle/c, OpenMP) for the same valid key, witness and (r, s) -- A, B, C byte for byte."""
    from oracle.c import run as oc
    cv = Conv("bn254")
    syn = syn20
    pk = syn.make_key()
    rng = random.Random(11)
    r_m, s_m = cv.fr([rng.randrange(cv.r)]), cv.fr([rng.randrange(cv.r)])
    A, Bp, Cp = pk.prove_plain(syn.public_inputs, syn.private_witness, r_m, s_m)
    desc, keep = oc.key_desc(syn.matrices, syn.points)
    a, b, c = oc.prove_plain(desc, syn.public_inputs, syn.private_witness, r_m, s_m)
    assert (A == a).all() and (Bp == b).all() and (Cp == c).all(), "GPU proof bytes differ from oracle/c at 2^20"
    # the witness map alone, all 2^20 half shares
    h_gpu = pk.witness_map(syn.public_inputs, syn.private_witness)
    h_cpu = oc.witness_map(desc, 0, 0, syn.public_inputs, syn.private_witness)
    assert (h_gpu == h_cpu).all()
    pk.free()
    del keep


def test_groth16_rep3_2p20_opens_to_oracle_c_proof(gpu_ctx, syn20):
    """The metric's own configuration (co-Groth16, 3-party Rep3, 2^20 constraints), three parties as threads on this
    GPU through the library's protocol (cs_groth16_rep3_prove over mailbox nets): every party returns the same
    proof, and it equals oracle/c's plain proof for r = sum r_i.a, s = sum s_i.a -- bit-exact at full size."""
    import threading
    from co_snarks_b200.rep3 import random_field_limbs
    from oracle.c import run as oc
    cv = Conv("bn254")
    syn = syn20
    lib = gpu_ctx.lib
    # replicated sharing of the witness (rep3.rs:281-293), vectorised: x = x0 + x1 + x2
    share_rng = np.random.Generator(np.random.PCG64(5))
    nw = syn.private_witness.shape[0]
    x0, x1 = random_field_limbs(share_rng, nw), random_field_limbs(share_rng, nw)
    d0, d1, dw = gpu_ctx.to_device(x0), gpu_ctx.to_device(x1), gpu_ctx.to_device(syn.private_witness)
    # shares are Montgomery representations: treat the random limbs as such and subtract on the device
    gpu_ctx._check(lib.cs_vec_sub(gpu_ctx.h, cv.id, dw, d0, dw, nw))
    gpu_ctx._check(lib.cs_vec_sub(gpu_ctx.h, cv.id, dw, d1, dw, nw))
    x2 = gpu_ctx.d2h(dw, (nw, 4))
    for d in (d0, d1, dw):
        gpu_ctx.free(d)
    xs = (x0, x1, x2)
    ctxs = [B.Context(0) for _ in range(3)]
    pks = [B.Groth16Key(c, B.CS_BN254, syn.matrices, syn.points) for c in ctxs]
    nets0 = [B.Net.peer(ctxs[i], i, 3) for i in range(3)]
    nets1 = [B.Net.peer(ctxs[i], i, 3) for i in range(3)]
    for i in range(3):
        nets0[i].connect_local(nets0)
        nets1[i].connect_local(nets1)
    seeds = [B.os_random(lib, 32) for _ in range(3)]
    states = [B.Rep3StateC.from_seeds(lib, i, seeds[i], seeds[(i + 2) % 3]) for i in range(3)]
    out, errs = {}, []

    def party(i):
        try:
            sh = np.ascontiguousarray(np.concatenate([xs[i], xs[(i + 2) % 3]], axis=1))
            out[i] = pks[i].rep3_prove(nets0[i], nets1[i], states[i], syn.public_inputs, sh, want_rs=True)
        except Exception as e:  # noqa: BLE001
            errs.append(e)
    th = [threading.Thread(target=party, args=(i,)) for i in range(3)]
    for t in th:
        t.start()
    for t in th:
        t.join(timeout=600)
    assert not errs, errs
    for i in (1, 2):
        assert all((out[i][k] == out[0][k]).all() for k in range(3)), "parties disagree on the proof"
    rs = [cv.fr_back(out[i][3]) for i in range(3)]
    r_tot = sum(x[0] for x in rs) % cv.r
    s_tot = sum(x[2] for x in rs) % cv.r
    desc, keep = oc.key_desc(syn.matrices, syn.points)
    a, b, c = oc.prove_plain(desc, syn.public_inputs, syn.private_witness, cv.fr([r_tot]), cv.fr([s_tot]))
    assert (out[0][0] == a).all() and (out[0][1] == b).all() and (out[0][2] == c).all(), \
        "opened Rep3 proof at 2^20 differs from oracle/c's plain proof for (sum r, sum s)"
    assert all(0 < n.bytes_sent < 2048 for n in nets0 + nets1)
    for pk in pks:
        pk.free()
    for n in nets0 + nets1:
        n.free()
    for c_ in ctxs:
        c_.close()
    del keep


def test_groth16_2p20_proof_verifies(gpu_ctx, syn20):
    cv = Conv("bn254")
    syn = syn20
    pk = syn.make_key()
    rng = random.Random(3)
    r_, s_ = rng.randrange(cv.r), rng.randrange(cv.r)
    A, Bp, Cp = pk.prove_plain(syn.public_inputs, syn.private_witness, cv.fr([r_]), cv.fr([s_]))
    proof = (cv.pt1(A), cv.pt2(Bp), cv.pt1(Cp))
    vk = syn.vk_ints()
    assert groth16_verify(vk, syn.witness[1:2], proof)
    assert not groth16_verify(vk, [(syn.witness[1] + 1) % cv.r], proof)
    # determinism: the same (r, s) gives the same bytes
    A2, B2, C2 = pk.prove_plain(syn.public_inputs, syn.private_witness, cv.fr([r_]), cv.fr([s_]))
    assert (A == A2).all() and (Bp == B2).all() and (Cp == C2).all()
    pk.free()


@pytest.mark.parametrize("lg,batch", [(22, 2), (24, 1)])
def test_ntt_plonk_sizes_roundtrip(gpu_ctx, lg, batch):
    """co-Plonk domain sizes (BASELINE configs[3]: n = 2^22, extended 4n = 2^24; Rep3 shares = batch 2): 3-pass
    transforms.  Every output of each direction, on its own input, of the natural-order transforms and of the bit
    reversal equals oracle/c's radix-2 loop (tests/test_production_shapes.py has the other pass splits); the round trip
    fft_out_to_in(ifft_in_to_out(x)) == x is kept as well."""
    K.check_ntt_against_oracle_c(gpu_ctx, "bn254", lg, batch)
    cv = Conv("bn254")
    n = 1 << lg
    g, _ = groth16_roots_of_unity(cv.r, lg)
    dom = gpu_ctx.domain(cv.id, lg, cv.fr([g]))
    a = _rand_fr_limbs(n * batch, 7 + lg, cv.r)
    da = gpu_ctx.to_device(a)
    dom.ifft_in_to_out(da, batch)
    dom.fft_out_to_in(da, batch)
    assert (gpu_ctx.d2h(da, (n * batch, 4)) == a).all()
    gpu_ctx.free(da)
    dom.free()


def test_plonk_synthetic_2p10_equals_oracle(gpu_ctx):
    K.check_plonk_synthetic(gpu_ctx, 10, n_public=3)


def test_plonk_synthetic_2p16_verifies(gpu_ctx):
    """A 2^16-gate proof (4n = 2^18-point quotient) checked by the oracle's pairing verifier."""
    K.check_plonk_synthetic(gpu_ctx, 16, n_public=2, against_oracle=False)
