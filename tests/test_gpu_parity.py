"""GPU parity tests (run with -m gpu on an H100): libcosnarks_gpu.so through the C ABI against
the oracle / golden vectors.  Bit-exact: all arithmetic is integer."""
import pytest

import kernel_checks as K

pytestmark = pytest.mark.gpu


def test_field_ops(gpu_ctx):
    K.check_field_ops(gpu_ctx, n=4099)


def test_share_kernels(gpu_ctx):
    K.check_share_kernels(gpu_ctx, n=3001)


def test_roots(gpu_ctx):
    K.check_roots(gpu_ctx)
    K.check_roots(gpu_ctx, "bls12_381")


def test_ntt_small(gpu_ctx):
    K.check_ntt(gpu_ctx, [0, 1, 2, 3, 7, 10, 11])


def test_ntt_multi_pass(gpu_ctx):
    K.check_ntt(gpu_ctx, [13, 14])


def test_msm_g1(gpu_ctx):
    K.check_msm(gpu_ctx, 0, 1500, window_bits=(0, 5, 11, 19))


def test_msm_g1_tiny(gpu_ctx):
    K.check_msm(gpu_ctx, 0, 3, window_bits=(0,))


def test_msm_g2(gpu_ctx):
    K.check_msm(gpu_ctx, 1, 300, window_bits=(0, 8, 18))


def test_msm_crs_points(gpu_ctx):
    K.check_msm_crs(gpu_ctx)


def test_fixed_base_mul(gpu_ctx):
    K.check_fixed_base_mul(gpu_ctx, n=70)


def test_plonk_round1_kat_bn254(gpu_ctx):
    K.check_plonk_round1_kat(gpu_ctx)


def test_groth16_multiplier2(gpu_ctx):
    K.check_groth16_fixture(gpu_ctx, "multiplier2")


def test_groth16_poseidon(gpu_ctx):
    K.check_groth16_fixture(gpu_ctx, "poseidon")


# ---- BLS12-381
def test_bls12_381_field_and_ntt(gpu_ctx):
    K.check_field_ops(gpu_ctx, n=1025, curve="bls12_381")
    K.check_ntt(gpu_ctx, [1, 6, 12], curve="bls12_381")


def test_bls12_381_msm_g1(gpu_ctx):
    K.check_msm(gpu_ctx, 0, 700, window_bits=(0, 9), curve="bls12_381")


def test_bls12_381_msm_g2(gpu_ctx):
    K.check_msm(gpu_ctx, 1, 150, curve="bls12_381")


def test_plonk_round1_kat_bls12_381(gpu_ctx):
    """4096-point iNTT + ~4100-point MSM on BLS12-381 == the reference's known answers (round1.rs:397-417)."""
    K.check_plonk_round1_kat(gpu_ctx, "bls12_381", "poseidon")


def test_msm_rep3_shares(gpu_ctx):
    K.check_msm_rep3_shares(gpu_ctx, n=900)


def test_groth16_shamir_local(gpu_ctx):
    K.check_groth16_shamir_local(gpu_ctx)


def test_plonk_primitives(gpu_ctx):
    K.check_plonk_primitives(gpu_ctx, lg=11)


def test_rep3_mask_prf(gpu_ctx):
    K.check_rep3_mask_prf(gpu_ctx, n=5000)


def test_shamir_degree_reduce(gpu_ctx):
    K.check_shamir_degree_reduce(gpu_ctx, n=3000)


def test_zkey_ingest(gpu_ctx, tmp_path):
    K.check_zkey_ingest(gpu_ctx, tmp_path, "poseidon")


def test_prove_cli(gpu_ctx, tmp_path):
    K.check_prove_cli(None, tmp_path, "poseidon")
    K.check_prove_cli_plonk(None, tmp_path, "multiplier2")


def test_libsnark_reduction(gpu_ctx):
    K.check_libsnark_reduction(gpu_ctx, m_vars=3000)


@pytest.mark.gpu
def test_rep3_mul_vec_reshare(gpu_ctx):
    K.check_rep3_mul_vec_reshare(gpu_ctx)


def test_keccak(gpu_ctx):
    K.check_keccak(gpu_ctx.lib)


def test_plonk_prove_multiplier2(gpu_ctx):
    K.check_plonk_prove(gpu_ctx, "multiplier2")


def test_plonk_prove_poseidon(gpu_ctx):
    K.check_plonk_prove(gpu_ctx, "poseidon")


def test_plonk_rep3_multiplier2(gpu_ctx):
    K.check_plonk_rep3(gpu_ctx, "multiplier2")


def test_plonk_rep3_poseidon(gpu_ctx):
    K.check_plonk_rep3(gpu_ctx, "poseidon")


def test_plonk_rep3_synthetic(gpu_ctx):
    K.check_plonk_rep3_synthetic(gpu_ctx, 9, n_public=3)


def test_plonk_prove_bls12_381(gpu_ctx):
    """The BLS12-381 instantiation (255-bit Fr, 6-limb Fq) on the reference's bls12_381/multiplier2 fixture."""
    K.check_plonk_prove(gpu_ctx, "multiplier2", curve="bls12_381")


def test_plonk_zkey_ingest(gpu_ctx, tmp_path):
    K.check_plonk_zkey_ingest(gpu_ctx, tmp_path, "multiplier2")
    K.check_plonk_zkey_ingest(gpu_ctx, tmp_path, "multiplier2", curve="bls12_381")


def test_crs_file_ingest(gpu_ctx, tmp_path):
    K.check_crs_file_ingest(gpu_ctx, tmp_path)


def test_groth16_bls12_381(gpu_ctx):
    """Groth16 on the BLS12-381 instantiation (6-limb Fq, 255-bit Fr) on the GPU: witness map + five MSMs + assembly on
    the reference's bls12_381/multiplier2 fixture; proof bytes == oracle, accepted by the BLS12-381 pairing check
    under the snarkjs verification key (the acceptance criterion of co-groth16/src/lib.rs:93-119)."""
    K.check_groth16_fixture(gpu_ctx, "multiplier2", curve="bls12_381")


def test_groth16_bls12_381_poseidon(gpu_ctx):
    """The reference's bls12_381/poseidon circuit on the GPU: witness map == golden h, proof bytes == the oracle's,
    accepted under the snarkjs key; the Rep3 local phases of three parties open to the plain proof."""
    K.check_groth16_fixture(gpu_ctx, "poseidon", curve="bls12_381")


@pytest.mark.parametrize("name", ["multiplier2", "poseidon"])
def test_groth16_shamir_local_bls12_381(gpu_ctx, name):
    K.check_groth16_shamir_local(gpu_ctx, name, curve="bls12_381")


def test_zkey_ingest_bls12_381(gpu_ctx, tmp_path):
    K.check_zkey_ingest(gpu_ctx, tmp_path, "poseidon", curve="bls12_381")


def test_msm_fp64_pipe_accumulation_subprocess():
    """The opt-in FP64-pipe bucket accumulation (cs_msm52.cuh, CS_MSM_F52=1: 5 x 52-bit limbs, DFMA split products,
    lazy ranges, exact-slice fallback for P + P / P + (-P)) gives the same bits as the oracle on the MSM edge-case
    suite.  Separate process: the switch is read once per process at the first base upload."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r);"
            "from co_snarks_b200 import binding as B; import kernel_checks as K;"
            "ctx = B.Context(0); K.check_msm(ctx, 0, 700, window_bits=(0, 9)); K.check_msm(ctx, 0, 5000); print('ok')"
            % (root, os.path.join(root, "tests")))
    env = dict(os.environ, CS_MSM_F52="1")
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "ok" in out.stdout, out.stdout + out.stderr


def test_ntt_tma_radix8_pass_subprocess():
    """The opt-in TMA-staged radix-8 NTT pass (cs_ntt8.cuh, CS_NTT_V2=1: cp.async.bulk tile loads with mbarrier,
    multi-column tiles, register radix-8/4 rounds) gives the oracle's transforms at every size it takes over (2^12 up),
    batch 1 and 2, forward / inverse, and through the Plonk fft/ifft entry points.  Separate process: the switch is
    read once per process."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r);"
            "from co_snarks_b200 import binding as B; import kernel_checks as K;"
            "ctx = B.Context(0); K.check_ntt(ctx, (12, 13, 14, 15)); K.check_plonk_primitives(ctx, lg=13); print('ok')"
            % (root, os.path.join(root, "tests")))
    env = dict(os.environ, CS_NTT_V2="1")
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and "ok" in out.stdout, out.stdout + out.stderr


def test_rep3_batch_vm_ops(gpu_ctx):
    K.check_rep3_batch_ops(gpu_ctx, n=3001)


def test_honk_commit_batch(gpu_ctx):
    K.check_honk_commit_batch(gpu_ctx, n=1000)


def test_share_rep3_device(gpu_ctx):
    K.check_share_rep3_device(gpu_ctx, n=100000)


def test_sumcheck_kernels(gpu_ctx):
    K.check_sumcheck(gpu_ctx, log_n=9)


def test_sumcheck_kernels_bls12_381(gpu_ctx):
    K.check_sumcheck(gpu_ctx, log_n=5, curve="bls12_381")
