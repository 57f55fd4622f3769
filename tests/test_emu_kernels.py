"""CPU-only: the exact device algorithms (csrc/*.cu compiled by tests/emu with -DCS_EMU) against the
oracle and the golden vectors, at sizes that finish in seconds.  This is host-side verification of
the kernels' logic; the GPU parity tests proper are tests/test_gpu_parity.py."""
import os

import pytest

import kernel_checks as K


def test_emu_field_ops(emu_ctx):
    K.check_field_ops(emu_ctx, n=97)


def test_emu_share_kernels(emu_ctx):
    K.check_share_kernels(emu_ctx, n=50)


def test_emu_roots(emu_ctx):
    K.check_roots(emu_ctx)
    K.check_roots(emu_ctx, "bls12_381")


def test_emu_ntt(emu_ctx):
    K.check_ntt(emu_ctx, [0, 1, 2, 5, 11])


def test_emu_msm_g1(emu_ctx):
    K.check_msm(emu_ctx, 0, 120, window_bits=(0, 7))


def test_emu_msm_g1_slice64(emu_ctx, monkeypatch):
    """the 64-entries-per-slice path used for windows >= 18 bits, forced on a small bucket count"""
    monkeypatch.setenv("CS_MSM_SLICE", "64")
    K.check_msm(emu_ctx, 0, 300, window_bits=(5,))


def test_emu_msm_g2(emu_ctx):
    K.check_msm(emu_ctx, 1, 40, window_bits=(0,))


def test_emu_fixed_base_mul(emu_ctx):
    K.check_fixed_base_mul(emu_ctx, n=6)


def test_emu_plonk_round1_kat(emu_ctx):
    K.check_plonk_round1_kat(emu_ctx)


def test_emu_groth16_multiplier2(emu_ctx):
    K.check_groth16_fixture(emu_ctx, "multiplier2")


# ---- BLS12-381 (12-limb Fq, 255-bit Fr)
def test_emu_bls12_381_field_and_ntt(emu_ctx):
    K.check_field_ops(emu_ctx, n=40, curve="bls12_381")
    K.check_ntt(emu_ctx, [1, 6], curve="bls12_381")


def test_emu_bls12_381_msm(emu_ctx):
    K.check_msm(emu_ctx, 0, 40, curve="bls12_381")
    K.check_msm(emu_ctx, 1, 14, curve="bls12_381")


def test_emu_msm_rep3_shares(emu_ctx):
    K.check_msm_rep3_shares(emu_ctx, n=60)


def test_emu_groth16_shamir_local(emu_ctx):
    K.check_groth16_shamir_local(emu_ctx)


def test_emu_plonk_primitives(emu_ctx):
    K.check_plonk_primitives(emu_ctx, lg=5)


def test_emu_rep3_mask_prf(emu_ctx):
    K.check_rep3_mask_prf(emu_ctx, n=40)


def test_emu_shamir_degree_reduce(emu_ctx):
    K.check_shamir_degree_reduce(emu_ctx, n=20)


def test_emu_zkey_ingest(emu_ctx, tmp_path):
    K.check_zkey_ingest(emu_ctx, tmp_path, "multiplier2")


def test_emu_prove_cli(emu_ctx, tmp_path):
    import os, sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "emu"))
    import build_emu
    K.check_prove_cli(build_emu.OUT, tmp_path)
    K.check_prove_cli_plonk(build_emu.OUT, tmp_path)
    K.check_prove_cli_rep3_shares(build_emu.OUT, tmp_path)


def test_emu_libsnark_reduction(emu_ctx):
    K.check_libsnark_reduction(emu_ctx, m_vars=20)


def test_rep3_mul_vec_reshare(emu_ctx):
    K.check_rep3_mul_vec_reshare(emu_ctx, use_ipc=True)


def test_keccak(emu_ctx):
    K.check_keccak(emu_ctx.lib)


def test_plonk_prove_multiplier2(emu_ctx):
    K.check_plonk_prove(emu_ctx, "multiplier2")


@pytest.mark.skipif(os.environ.get("CS_FULL_CPU_TESTS", "0") != "1",
                    reason="one minute under emulation; the same check runs on the GPU (tests/test_gpu_parity.py) -- "
                           "set CS_FULL_CPU_TESTS=1 to run it here")
def test_plonk_prove_poseidon(emu_ctx):
    K.check_plonk_prove(emu_ctx, "poseidon", random_blinders=False)


def test_plonk_synthetic_key(emu_ctx):
    K.check_plonk_synthetic(emu_ctx, 5, n_public=2)
    K.check_plonk_synthetic(emu_ctx, 4, n_public=0)


def test_plonk_rep3_multiplier2(emu_ctx):
    K.check_plonk_rep3(emu_ctx, "multiplier2")
    K.check_plonk_rep3_drawn_blinders(emu_ctx, "multiplier2")


def test_plonk_rep3_synthetic(emu_ctx):
    K.check_plonk_rep3_synthetic(emu_ctx, 4, n_public=2)


def test_plonk_key_errors(emu_ctx):
    K.check_plonk_key_errors(emu_ctx)


def test_plonk_prove_bls12_381(emu_ctx):
    """The BLS12-381 instantiation (255-bit Fr, 6-limb Fq) on the reference's bls12_381/multiplier2 fixture."""
    K.check_plonk_prove(emu_ctx, "multiplier2", curve="bls12_381")


def test_plonk_zkey_ingest(emu_ctx, tmp_path):
    K.check_plonk_zkey_ingest(emu_ctx, tmp_path, "multiplier2")
    K.check_plonk_zkey_ingest(emu_ctx, tmp_path, "multiplier2", curve="bls12_381")


def test_crs_file_ingest(emu_ctx, tmp_path):
    K.check_crs_file_ingest(emu_ctx, tmp_path)


def test_emu_groth16_bls12_381(emu_ctx):
    """Groth16 on BLS12-381 (6-limb Fq, 255-bit Fr): witness map and proof bytes == oracle on the reference's
    bls12_381/multiplier2 fixture, proof accepted by the BLS12-381 pairing check under the snarkjs key."""
    K.check_groth16_fixture(emu_ctx, "multiplier2", curve="bls12_381")


def test_emu_groth16_bls12_381_poseidon(emu_ctx):
    """The reference's bls12_381/poseidon circuit: witness map == golden h, proof bytes == the oracle's, and the Rep3
    local phases of three parties open to the plain proof."""
    K.check_groth16_fixture(emu_ctx, "poseidon", curve="bls12_381")


@pytest.mark.parametrize("name", ["multiplier2", "poseidon"])
def test_emu_groth16_shamir_local_bls12_381(emu_ctx, name):
    K.check_groth16_shamir_local(emu_ctx, name, curve="bls12_381")


def test_emu_zkey_ingest_bls12_381(emu_ctx, tmp_path):
    K.check_zkey_ingest(emu_ctx, tmp_path, "poseidon", curve="bls12_381")


def test_emu_rep3_batch_vm_ops(emu_ctx):
    K.check_rep3_batch_ops(emu_ctx, n=33)


def test_emu_honk_commit_batch(emu_ctx):
    K.check_honk_commit_batch(emu_ctx, n=40)


def test_emu_share_rep3_device(emu_ctx):
    K.check_share_rep3_device(emu_ctx, n=60)


def test_rep3_share_files(emu_ctx, tmp_path):
    K.check_rep3_share_files(emu_ctx.lib, tmp_path)


def test_emu_sumcheck(emu_ctx):
    K.check_sumcheck(emu_ctx, log_n=4)


def test_emu_sumcheck_bls12_381(emu_ctx):
    K.check_sumcheck(emu_ctx, log_n=3, curve="bls12_381")
