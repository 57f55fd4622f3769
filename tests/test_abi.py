"""CPU-only: the C-ABI library loads, exports every symbol include/cosnarks_gpu.h declares, binds them in
co_snarks_b200/binding.py, and FAILS LOUDLY without a GPU (no CPU fallback)."""
import os
import re

import pytest

from co_snarks_b200 import binding as B

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    src = open(os.path.join(ROOT, "include", "cosnarks_gpu.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(cs_[a-z0-9_]+)\s*\(", src)))


def test_header_declares_and_library_exports_every_symbol():
    lib = B.load()
    syms = header_symbols()
    assert len(syms) >= 40
    for s in syms:
        assert hasattr(lib, s), "libcosnarks_gpu.so does not export " + s
        assert s in B.SIGNATURES, "binding.py has no signature for " + s
    for s in B.SIGNATURES:
        assert s in syms, "binding.py binds %s which the header does not declare" % s


def test_version_string():
    lib = B.load()
    assert b"sm_90a" in lib.cs_version()


def test_no_cpu_fallback_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    with pytest.raises(B.CsError) as e:
        B.Context(0)
    assert "no CUDA device" in str(e.value) or "CUDA error" in str(e.value)


def test_host_helpers_work_without_gpu():
    """Single-point helpers and Montgomery conversion run on the host inside the library."""
    from helpers import Conv
    from oracle.ec import g1
    from oracle.fields import BN254, groth16_roots_of_unity
    lib = B.load()
    cv = Conv("bn254")
    G = g1(BN254)
    P = G.mul(BN254.g1, 1234567)
    k = 987654321987654321
    out = B.point_scalar_mul(lib, cv.id, B.CS_G1, cv.g1([P])[0], cv.fr([k])[0])
    assert cv.pt1(out) == G.mul(P, k)
    out = B.point_add(lib, cv.id, B.CS_G1, cv.g1([P])[0], cv.g1([G.neg(P)])[0])
    assert cv.pt1(out) is None
    out = B.point_add(lib, cv.id, B.CS_G1, cv.g1([P])[0], cv.g1([P])[0])
    assert cv.pt1(out) == G.mul(P, 2)
    import numpy as np
    gen = np.zeros(4, dtype=np.uint64)
    shift = np.zeros(4, dtype=np.uint64)
    assert lib.cs_groth16_roots_of_unity(cv.id, 20, B._ptr(gen), B._ptr(shift)) == 0
    eg, es = groth16_roots_of_unity(cv.r, 20)
    assert cv.fr_back(gen) == [eg] and cv.fr_back(shift) == [es]
    assert lib.cs_groth16_roots_of_unity(cv.id, 29, B._ptr(gen), B._ptr(shift)) != 0
    assert b"Polynomial Degree too large" in lib.cs_last_error()


def test_argument_errors_come_back_as_codes_not_crashes():
    """Every entry point validates its arguments before touching CUDA: NULL handles / buffers give a negative
    code and a message through cs_last_error (no panics across the boundary, SURVEY 8b)."""
    import ctypes as C
    import numpy as np
    lib = B.load()
    null = None
    out = C.c_void_p()
    calls = [
        lambda: lib.cs_plonk_pk_create(null, null, C.byref(out)),
        lambda: lib.cs_plonk_pk_from_zkey(null, b"/nonexistent.zkey", C.byref(out), null, null),
        lambda: lib.cs_plonk_prove_plain(null, null, null, 0, null, 0, null, null, null),
        lambda: lib.cs_plonk_rep3_create(null, null, 0, C.byref(out)),
        lambda: lib.cs_plonk_rep3_step(null, 1, null, null),
        lambda: lib.cs_plonk_rep3_round1(null, null, null, 0, null, 0, null, null),
        lambda: lib.cs_rep3_mul_vec_reshare(null, 0, null, null, 4, null, null, null),
        lambda: lib.cs_ipc_export(null, null, null),
        lambda: lib.cs_bases_from_crs_file(null, b"/nonexistent.dat", 0, 4, 0, C.byref(out)),
        lambda: lib.cs_groth16_pk_from_zkey(null, b"/nonexistent.zkey", 0, C.byref(out), null),
        lambda: lib.cs_msm(null, null, 0, null, 4, 1, null, null),
        lambda: lib.cs_plonk_pk_info(null, null, null, null, null),
        # round 2: transport, states, in-library parties, VM / Honk / sumcheck entry points
        lambda: lib.cs_net_send(null, 1, null, 0),
        lambda: lib.cs_net_sendrecv(null, 1, null, 0, 2, null, 0),
        lambda: lib.cs_net_peer_create(null, 0, 3, C.byref(out)),
        lambda: lib.cs_rep3_state_create(null, C.byref(out)),
        lambda: lib.cs_groth16_rep3_prove(null, null, null, null, null, null, null, null, null, null, null, null),
        lambda: lib.cs_groth16_shamir_prove(null, null, null, null, 3, 1, null, null, null, null, null, null),
        lambda: lib.cs_plonk_rep3_prove(null, null, null, null, 0, null, 0, null, null, null),
        lambda: lib.cs_plonk_rep3_connect_io(null, null, null),
        lambda: lib.cs_rep3_batch(null, 0, 0, 0, null, null, null, 4),
        lambda: lib.cs_honk_commit_batch(null, null, 0, null, null, 1, null),
        lambda: lib.cs_sumcheck_gate_separator(null, 0, null, 3, null),
        lambda: lib.cs_sumcheck_fold(null, 0, null, null, 1, 0, 4, null),
        lambda: lib.cs_sumcheck_arith_round(null, 0, 0, 0, null, 4, null, 2, null, null, null),
        lambda: lib.cs_shamir_state_create(null, 0, 3, 1, 0, C.byref(out)),
        lambda: lib.cs_rep3_witness_read(b"/nonexistent.shares", 0, null, 0, null, 0, null, null, null),
    ]
    for i, call in enumerate(calls):
        assert call() < 0, "call %d accepted NULL arguments" % i
        assert len(lib.cs_last_error()) > 0
    d = np.zeros(32, dtype=np.uint8)
    assert lib.cs_keccak256(b"abc", 3, B._ptr(d)) == 0
    assert bytes(d).hex() == "4e03657aea45a94fc7d47ba826c8d667c0d1e6e33a64a036ec44f58fa12d6c45"  # Keccak-256("abc")
