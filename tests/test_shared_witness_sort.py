"""One sort of the witness digits for Groth16's A, B1, B2 and L MSMs (cs_msm.cuh msm_view, cs_groth16.cu
plan_witness_views).

CPU, on the emulated kernels: the filtered view of the unmasked sort holds exactly the entries of the table's own
masked sort, bucket by bucket (an infinity entry kept or a finite one dropped changes a bucket count); and proofs equal
the oracle's for keys that make every kind of consumer occur -- A and B masks sparse and different, L with an infinite
base (an unused variable), a query whose witness range is entirely at infinity, no witness at all -- through the plain
prover, Rep3 with three party threads, and the two-GPU Rep3 split ({A, B1, L} on the protocol GPU, {H, B2} on the
helper).  GPU: the same proofs on the device.
"""
import ctypes
import os
import random
import subprocess
import sys
import threading

import numpy as np
import pytest

from co_snarks_b200 import binding as B
from helpers import Conv
from oracle import groth16 as OG
from workloads.synth_groth16 import SynthGroth16

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def _emu_lib():
    sys.path.insert(0, os.path.join(HERE, "emu"))
    import build_emu
    return build_emu.build()


def _emu_ctx():
    return B.Context(0, lib_path=_emu_lib())


# ---------------------------------------------------------------------------------------------- R1CS shapes
# rows as lists of (coeff, variable); variables 0 = one, 1 = public input
def _unused_variable():
    # a * b = c;  (c + x) * 1 = d;  u (variable 5) occurs in no constraint: A, B and L are infinite there
    x, a, b, u = 7, 3, 11, 5
    c = a * b
    w = [1, x, a, b, c, u, c + x]
    return ([[(1, 2)], [(1, 4), (1, 1)]], [[(1, 3)], [(1, 0)]], [[(1, 4)], [(1, 6)]], w, 2)


def _b_public_only():
    # (a + b) * x = c;  c * 1 = c: B uses public variables only, so B1 / B2 are infinite over the whole witness range
    x, a, b = 9, 4, 13
    return ([[(1, 2), (1, 3)], [(1, 4)]], [[(1, 1)], [(1, 0)]], [[(1, 4)], [(1, 4)]], [1, x, a, b, (a + b) * x], 2)


def _no_witness():
    # x * 1 = x with x public: nw = 0
    return ([[(1, 1)]], [[(1, 0)]], [[(1, 1)]], [1, 12345], 2)


SHAPES = {"synthetic_2p5": None, "unused_variable": _unused_variable, "b_public_only": _b_public_only,
          "no_witness": _no_witness}


def _synth(ctx, shape):
    f = SHAPES[shape]
    return SynthGroth16(ctx, 5) if f is None else SynthGroth16(ctx, 0, r1cs=f())


def _oracle_key(cv, syn):
    """The synthetic key and system in the oracle's conventions."""
    p = syn.points
    z = dict(curve=cv.c, alpha_g1=cv.pt1(p["alpha_g1"][0]), beta_g1=cv.pt1(p["beta_g1"][0]),
             delta_g1=cv.pt1(p["delta_g1"][0]), beta_g2=cv.pt2(p["beta_g2"][0]), delta_g2=cv.pt2(p["delta_g2"][0]))
    for k in ("a_query", "b_g1_query", "l_query", "h_query"):
        z[k] = [cv.pt1(row) for row in p[k]]
    z["b_g2_query"] = [cv.pt2(row) for row in p["b_g2_query"]]
    m = dict(num_constraints=syn.nc, num_instance_variables=syn.ni, num_witness_variables=syn.m - syn.ni,
             a=syn.a_rows, b=syn.b_rows)
    return z, m


def _check_masks(cv, syn, shape):
    """The key has the infinity pattern the case is about."""
    z, _ = _oracle_key(cv, syn)
    ni = syn.ni
    a_inf = [P is None for P in z["a_query"][ni:]]
    b_inf = [P is None for P in z["b_g1_query"][ni:]]
    assert b_inf == [P is None for P in z["b_g2_query"][ni:]]
    l_inf = [P is None for P in z["l_query"]]
    if shape == "synthetic_2p5":
        assert any(a_inf) and any(b_inf) and a_inf != b_inf and not any(l_inf)
    elif shape == "unused_variable":
        assert l_inf[5 - ni] and a_inf[5 - ni] and b_inf[5 - ni] and sum(l_inf) == 1
    elif shape == "b_public_only":
        assert all(b_inf) and not all(a_inf)
    else:
        assert syn.m == ni


def _prove_plain(ctx, shape, seed=11):
    cv = Conv("bn254")
    syn = _synth(ctx, shape)
    _check_masks(cv, syn, shape)
    pk = syn.make_key()
    rng = random.Random(seed)
    r_, s_ = rng.randrange(cv.r), rng.randrange(cv.r)
    A, Bp, Cp = pk.prove_plain(syn.public_inputs, syn.private_witness, cv.fr([r_]), cv.fr([s_]))
    pk.free()
    z, m = _oracle_key(cv, syn)
    assert (cv.pt1(A), cv.pt2(Bp), cv.pt1(Cp)) == OG.prove_plain(z, m, syn.witness, r_, s_)


def _shares(cv, syn, party, seed=5):
    wsh = OG.share_rep3(syn.witness[syn.ni:], cv.r, random.Random(seed))
    return cv.fr([x for ab in wsh[party] for x in ab]).reshape(-1, 8)


def _prove_rep3_threads(ctx_factory, shape, two_gpus=False):
    """Three party threads (and, with two_gpus, a helper thread per party holding {H, B2}); the opened proof must
    equal the oracle's plain proof for r = sum r_i.a, s = sum s_i.a."""
    cv = Conv("bn254")
    syn = _synth(ctx_factory(), shape)
    z, m = _oracle_key(cv, syn)
    pub = syn.public_inputs
    roles = 2 if two_gpus else 1
    ctxs = [[ctx_factory() for _ in range(roles)] for _ in range(3)]
    lib = ctxs[0][0].lib
    pks = [[B.Groth16Key(c, B.CS_BN254, syn.matrices, syn.points) for c in row] for row in ctxs]
    nets0 = [B.Net.peer(ctxs[i][0], i, 3) for i in range(3)]
    nets1 = [B.Net.peer(ctxs[i][0], i, 3) for i in range(3)]
    for i in range(3):
        nets0[i].connect_local(nets0)
        nets1[i].connect_local(nets1)
    pairs = None
    if two_gpus:
        pairs = [[B.Net.peer(ctxs[i][ro], ro, 2) for ro in range(2)] for i in range(3)]
        for i in range(3):
            for ro in range(2):
                pairs[i][ro].connect_local(pairs[i])
    seeds = [bytes([29 * (i + 1) + k for k in range(32)]) for i in range(3)]
    states = [B.Rep3StateC.from_seeds(lib, i, seeds[i], seeds[(i + 2) % 3]) for i in range(3)]
    clones = [s.clone() for s in states] if two_gpus else None
    out, errs = [], []

    def party(i):
        try:
            A, Bp, Cp, rs = pks[i][0].rep3_prove(nets0[i], nets1[i], states[i], pub, _shares(cv, syn, i),
                                                 pair=pairs[i][0] if two_gpus else None, want_rs=True)
            out.append((i, cv.pt1(A), cv.pt2(Bp), cv.pt1(Cp), cv.fr_back(rs)))
        except Exception as e:  # noqa: BLE001
            errs.append(e)

    def helper(i):
        try:
            pks[i][1].rep3_prove_helper(i, pairs[i][1], clones[i], pub, _shares(cv, syn, i))
        except Exception as e:  # noqa: BLE001
            errs.append(e)

    th = [threading.Thread(target=party, args=(i,)) for i in range(3)]
    if two_gpus:
        th += [threading.Thread(target=helper, args=(i,)) for i in range(3)]
    for t in th:
        t.start()
    for t in th:
        t.join(timeout=600)
    assert not errs, errs
    res = sorted(out)
    proofs = [(a, b, c) for _, a, b, c, _ in res]
    assert proofs[0] == proofs[1] == proofs[2], "parties disagree on the proof"
    r_tot = sum(x[4][0] for x in res) % cv.r
    s_tot = sum(x[4][2] for x in res) % cv.r
    assert proofs[0] == OG.prove_plain(z, m, syn.witness, r_tot, s_tot)
    for row in pks:
        for pk in row:
            pk.free()
    for n in nets0 + nets1 + ([p for row in pairs for p in row] if pairs else []):
        n.free()
    for s in states + (clones or []):
        s.free()


# ---------------------------------------------------------------------------------------------- the view itself
@pytest.fixture(scope="module")
def view_shim(tmp_path_factory):
    emu = _emu_lib()
    out = str(tmp_path_factory.mktemp("view_shim") / "libview_shim.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-DCS_EMU", "-DCS_ENABLE_BLS12_381", "-fPIC", "-shared", "-w",
                           "-I", os.path.join(HERE, "emu"), "-I", os.path.join(ROOT, "co_snarks_b200", "csrc"),
                           "-o", out, os.path.join(HERE, "emu", "view_shim.cpp"), emu,
                           "-Wl,-rpath," + os.path.dirname(emu)])
    return ctypes.CDLL(out)


def _buckets(arr, nb1):
    """count[] + entries -> {bucket: sorted entries}"""
    count = arr[:nb1]
    pos, out = nb1, {}
    for b in range(nb1):
        out[b] = sorted(arr[pos:pos + count[b]].tolist())
        pos += count[b]
    return count, out


@pytest.mark.parametrize("case", ["sparse_offset", "one_infinite_no_offset", "all_infinite", "none_infinite_offset"])
def test_view_equals_the_masked_sort_emu(view_shim, case):
    rng = random.Random(case)
    r = Conv("bn254").r
    n, c = 61, 4
    # a mix of full-size, small (many zero digits) and zero scalars
    scal = [rng.randrange(r) for _ in range(n - 20)] + [rng.randrange(1 << 12) for _ in range(15)] + [0] * 5
    rng.shuffle(scal)
    offset, nbases = {"sparse_offset": (3, n + 5), "one_infinite_no_offset": (0, n), "all_infinite": (2, n + 2),
                      "none_infinite_offset": (2, n + 2)}[case]
    inf = {"sparse_offset": [rng.random() < 0.4 for _ in range(nbases)],
           "one_infinite_no_offset": [i == 17 for i in range(nbases)],
           "all_infinite": [True] * nbases, "none_infinite_offset": [False] * nbases}[case]
    words = np.zeros((nbases + 31) // 32, dtype=np.uint32)
    for i, f in enumerate(inf):
        if f:
            words[i >> 5] |= np.uint32(1 << (i & 31))
    limbs = np.ascontiguousarray(B.ints_to_limbs(scal, 4)).view(np.uint32).reshape(n, 8)
    W = (254 + 1 + c - 1) // c
    nb1 = (1 << (c - 1)) + 1
    masked = np.zeros(nb1 + W * n, dtype=np.uint32)
    view = np.zeros(nb1 + W * n, dtype=np.uint32)
    p = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_uint32))  # noqa: E731
    assert view_shim.view_vs_masked(n, p(limbs), c, nbases, offset, p(words), p(masked), p(view)) == 0
    cm, bm = _buckets(masked, nb1)
    cv_, bv = _buckets(view, nb1)
    assert cv_.tolist() == cm.tolist(), "bucket counts differ: the view kept an infinity entry or dropped a finite one"
    assert bv == bm
    total = int(cm.sum())
    finite = sum(1 for i in range(n) if not inf[offset + i] and scal[i])
    assert (total == 0) == (finite == 0)
    # every entry is a slot of a finite base of this table
    for b in range(1, nb1):
        for e in bv[b]:
            slot = e & 0x7FFFFFFF
            assert slot % nbases >= offset and not inf[slot % nbases]


# ---------------------------------------------------------------------------------------------- proofs (CPU)
@pytest.mark.parametrize("shape", list(SHAPES))
def test_plain_proof_equals_oracle_emu(shape):
    _prove_plain(_emu_ctx(), shape)


@pytest.mark.parametrize("shape", ["synthetic_2p5", "unused_variable", "b_public_only"])
def test_rep3_three_threads_emu(shape):
    _prove_rep3_threads(_emu_ctx, shape)


@pytest.mark.parametrize("shape", ["synthetic_2p5", "unused_variable", "b_public_only"])
def test_rep3_two_gpus_per_party_split_emu(shape):
    _prove_rep3_threads(_emu_ctx, shape, two_gpus=True)


# ---------------------------------------------------------------------------------------------- proofs (GPU)
@pytest.mark.gpu
@pytest.mark.parametrize("shape", list(SHAPES))
def test_plain_proof_equals_oracle_gpu(gpu_ctx, shape):
    _prove_plain(gpu_ctx, shape)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["synthetic_2p5", "unused_variable"])
def test_rep3_three_threads_gpu(shape):
    _prove_rep3_threads(lambda: B.Context(0), shape)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["synthetic_2p5", "unused_variable"])
def test_rep3_two_gpus_per_party_split_gpu(shape):
    _prove_rep3_threads(lambda: B.Context(0), shape, two_gpus=True)
