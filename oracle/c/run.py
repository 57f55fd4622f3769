"""ctypes front-end of oracle/c/liboracle.so (oracle; test infrastructure / CPU baseline only)."""
import ctypes as C
import os
import subprocess
import time

import numpy as np

os.environ.setdefault("OMP_WAIT_POLICY", "PASSIVE")  # idle workers sleep: shared hosts may cap the CPU quota
HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "liboracle.so")
_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB):
            subprocess.check_call(["make", "-s", "-C", HERE])
        _lib = C.CDLL(LIB)
        _lib.oracle_num_threads.restype = C.c_int
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def msm(points_mont, scalars_mont, group=0):
    L = lib()
    points_mont = np.ascontiguousarray(points_mont, dtype=np.uint64)
    scalars_mont = np.ascontiguousarray(scalars_mont, dtype=np.uint64)
    out = np.zeros(8 if group == 0 else 16, dtype=np.uint64)
    fn = L.oracle_msm_g1 if group == 0 else L.oracle_msm_g2
    fn(_p(points_mont), _p(scalars_mont), C.c_size_t(4), C.c_size_t(scalars_mont.shape[0]), _p(out))
    return out


def ifft_in_to_out(data, lg, batch, gen_mont, curve=0):
    """In place on a contiguous np.uint64 array of Montgomery Fr elements; curve = cs_curve id (0 BN254, 1 BLS12-381)."""
    assert data.flags.c_contiguous and data.dtype == np.uint64
    rc = lib().oracle_ifft_in_to_out(_p(data), C.c_uint(lg), C.c_uint(batch), _p(np.ascontiguousarray(gen_mont)), C.c_int(curve))
    assert rc == 0, "oracle_ifft_in_to_out: unknown curve %d" % curve
    return data


def fft_out_to_in(data, lg, batch, gen_mont, curve=0):
    assert data.flags.c_contiguous and data.dtype == np.uint64
    rc = lib().oracle_fft_out_to_in(_p(data), C.c_uint(lg), C.c_uint(batch), _p(np.ascontiguousarray(gen_mont)), C.c_int(curve))
    assert rc == 0, "oracle_fft_out_to_in: unknown curve %d" % curve
    return data


def key_desc(matrices_csr, points, curve=0):
    """Same descriptor as co_snarks_b200.binding.KeyDesc (include/cosnarks_gpu.h: cs_groth16_key_desc).  curve = cs_curve
    id: the witness map follows it (BN254 or BLS12-381 Fr); prove_plain takes BN254 keys only."""
    from co_snarks_b200.binding import KeyDesc, u32p, u64p  # type definition only
    d = KeyDesc()
    keep = []
    d.curve = curve
    d.num_constraints = matrices_csr["num_constraints"]
    d.num_instance_variables = matrices_csr["num_instance_variables"]
    d.num_witness_variables = matrices_csr["num_witness_variables"]
    for name in ("a", "b"):
        rp, col, coeff = (np.ascontiguousarray(x) for x in matrices_csr[name])
        keep += [rp, col, coeff]
        setattr(d, name + "_row_ptr", rp.ctypes.data_as(u32p))
        setattr(d, name + "_col", col.ctypes.data_as(u32p))
        setattr(d, name + "_coeff", coeff.ctypes.data_as(u64p))
        setattr(d, name + "_nnz", col.shape[0])
    for name in ("alpha_g1", "beta_g1", "beta_g2", "delta_g1", "delta_g2", "a_query", "b_g1_query", "b_g2_query",
                 "l_query", "h_query"):
        arr = np.ascontiguousarray(points[name], dtype=np.uint64)
        keep.append(arr)
        setattr(d, name, arr.ctypes.data_as(u64p))
        if name.endswith("query"):
            setattr(d, name + "_len", arr.shape[0])
    return d, keep


def witness_map(desc, kind, party, pub, wit, m1=None, m2=None):
    n = 1
    while n < desc.num_constraints + desc.num_instance_variables:
        n <<= 1
    out = np.zeros((n, 4), dtype=np.uint64)
    rc = lib().oracle_witness_map(C.byref(desc), kind, party, _p(pub), _p(wit), _p(m1), _p(m2), _p(out))
    assert rc == 0, "oracle_witness_map: unknown curve %d or domain beyond its two-adicity" % desc.curve
    return out


def prove_plain(desc, pub, wit, r_m, s_m):
    a = np.zeros(8, dtype=np.uint64)
    b = np.zeros(16, dtype=np.uint64)
    c = np.zeros(8, dtype=np.uint64)
    rc = lib().oracle_groth16_prove_plain(C.byref(desc), _p(pub), _p(wit), _p(r_m), _p(s_m), _p(a), _p(b), _p(c))
    assert rc == 0
    return a, b, c


# ------------------------------------------------------------------------------------------ bench legs
def _workload(log_m):
    """Synthetic R1CS + key for the CPU legs.  The CPU run needs no valid key (timing only), so the
    query points are i*G built by repeated addition on the host -- no GPU involved."""
    from workloads.synth_groth16 import make_r1cs, BN254_R, _fr
    m = 1 << log_m
    a_rows, b_rows, _, w = make_r1cs(m, 1)

    def csr(rows):
        rp = np.zeros(len(rows) + 1, dtype=np.uint32)
        cols, cfs = [], []
        for i, row in enumerate(rows):
            for cf, v in row:
                cols.append(v)
                cfs.append(cf)
            rp[i + 1] = len(cols)
        return rp, np.array(cols, dtype=np.uint32), _fr(cfs)

    mats = dict(num_constraints=m - 2, num_instance_variables=2, num_witness_variables=m - 2, a=csr(a_rows), b=csr(b_rows))
    return mats, _fr(w[:2]), _fr(w[2:]), m


def _points_by_addition(n, group):
    """n distinct curve points (k*G, k = 1..n) produced by the C library's own msm of unit vectors would
    be circular; instead use the affine chain P_{k+1} = P_k + G computed with python ints."""
    from oracle.fields import BN254
    from oracle.ec import g1, g2
    from co_snarks_b200.binding import ints_to_limbs, to_mont_ints
    G = g1(BN254) if group == 0 else g2(BN254)
    gen = BN254.g1 if group == 0 else BN254.g2
    # a short chain is tiled: distinctness of bases does not matter for CPU timing
    base = []
    P = gen
    for _ in range(min(n, 2048)):
        base.append(P)
        P = G.add(P, gen)
    flat = []
    for P in base:
        flat += [P[0], P[1]] if group == 0 else [P[0][0], P[0][1], P[1][0], P[1][1]]
    arr = ints_to_limbs(to_mont_ints(flat, BN254.q, 4), 4).reshape(len(base), -1)
    reps = (n + len(base) - 1) // len(base)
    return np.tile(arr, (reps, 1))[:n].copy()


def _timing_key(mats, m):
    """Timing-only key with the VALID key's sparsity: in a real (and in the synthetic valid) Groth16 key the B-query
    entry of a variable that occurs in no B row is the point at infinity (B_i(tau) = 0; 37 % of this workload's
    variables), and both provers skip those bases -- so the CPU arm must see the same infinity pattern as the GPU
    arm to do the same MSM work.  Point VALUES do not matter for CPU timing; they are k*G by repeated addition."""
    g1p = _points_by_addition(m, 0)
    g2p = _points_by_addition(m, 1)
    in_b = np.zeros(m, dtype=bool)
    in_b[mats["b"][1]] = True
    b1, b2 = g1p.copy(), g2p.copy()
    b1[~in_b] = 0
    b2[~in_b] = 0
    pts = dict(alpha_g1=g1p[:1], beta_g1=g1p[1:2], beta_g2=g2p[:1], delta_g1=g1p[2:3], delta_g2=g2p[1:2],
               a_query=g1p, b_g1_query=b1, b_g2_query=b2, l_query=g1p[:m - 2], h_query=g1p)
    return pts, float((~in_b).mean())


def time_proof(log_m, steps=1, warmup=0, budget_s=None):
    """-> (seconds per proof, steps actually timed, fraction of B-query bases at infinity).  budget_s bounds the
    whole call: the step count is cut (never below 1) when the first proof shows that `steps` would not fit."""
    mats, pub, wit, m = _workload(log_m)
    pts, inf_frac = _timing_key(mats, m)
    desc, keep = key_desc(mats, pts)
    from workloads.synth_groth16 import _fr
    r_m, s_m = _fr([123456789]), _fr([987654321])
    t0 = time.perf_counter()
    for _ in range(max(warmup, 0)):
        prove_plain(desc, pub, wit, r_m, s_m)
        if budget_s and time.perf_counter() - t0 > budget_s / 4:
            break
    t1 = time.perf_counter()
    done = 0
    for _ in range(steps):
        prove_plain(desc, pub, wit, r_m, s_m)
        done += 1
        if budget_s and done < steps:
            per = (time.perf_counter() - t1) / done
            if (time.perf_counter() - t0) + per > budget_s:
                break
    dt = (time.perf_counter() - t1) / done
    del keep
    return dt, done, inf_frac


def tune_threads(probe_log_m=15):
    """The reference's rayon pool uses every core it sees; on a shared box the visible core count can
    exceed the CPU quota, so pick the thread count that is fastest on a small proof."""
    L = lib()
    mx = os.cpu_count() or L.oracle_num_threads()
    best, best_t = mx, None
    cands = sorted({mx, max(1, mx // 2), max(1, mx // 4), max(1, mx // 8)}, reverse=True)
    mats, pub, wit, m = _workload(probe_log_m)
    pts, _ = _timing_key(mats, m)
    desc, keep = key_desc(mats, pts)
    from workloads.synth_groth16 import _fr
    r_m, s_m = _fr([3]), _fr([5])
    for t in cands:
        L.oracle_set_threads(t)
        prove_plain(desc, pub, wit, r_m, s_m)
        t0 = time.perf_counter()
        prove_plain(desc, pub, wit, r_m, s_m)
        dt = time.perf_counter() - t0
        if best_t is None or dt < best_t:
            best, best_t = t, dt
    L.oracle_set_threads(best)
    del keep
    return best


def cpu_baseline(log_m=20, target_log_m=20):
    cores = tune_threads()
    dt, done, inf_frac = time_proof(log_m, steps=2, warmup=1, budget_s=30)
    scale = (1 << target_log_m) / (1 << log_m)
    return {"value": 1.0 / (dt * scale), "unit": "proofs/s", "cores": int(cores), "kind": "port",
            "sample": "%d full Groth16 proof(s) at 2^%d constraints by oracle/c (OpenMP, %d threads) after 1 warm-up, %.2f s "
                      "each; same R1CS and the valid key's infinity pattern (%.0f %% of the B-query bases)%s" % (
                done, log_m, cores, dt, 100 * inf_frac, "" if scale == 1 else "; scaled linearly x%g to 2^%d" % (scale, target_log_m)),
            "seconds_per_proof": dt * scale}


def reference_arm(log_m=20, target_log_m=20, steps=1, warmup=0):
    """bench.py --impl reference: the reference's CPU path as restated by oracle/c (the Rust reference
    cannot be built here: no cargo, crates not vendored), all host threads."""
    cores = tune_threads()
    want = max(1, steps)
    dt, done, inf_frac = time_proof(log_m, steps=want, warmup=warmup, budget_s=170)
    scale = (1 << target_log_m) / (1 << log_m)
    v = 1.0 / (dt * scale)
    sample = "%d Groth16 proof(s) at 2^%d constraints (of %d requested; the run is bounded to ~3 minutes), oracle/c OpenMP " \
             "port on %d host threads" % (done, log_m, want, cores)
    return {"impl": "reference", "metric": "co-Groth16 proofs/sec (BN254, 2^20 constraints); MSM Mscalar/s",
            "value": v, "unit": "proofs/s", "n_gpus": 0, "steps": done, "warmup": warmup,
            "ms_per_step": dt * scale * 1e3, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": "u64x4 (256-bit Montgomery, integer)",
            "data": "synthetic (same seeded R1CS as the GPU arm; timing-only key with the valid key's infinity pattern: "
                    "%.0f %% of the B-query bases are the point at infinity and are skipped by both arms)" % (100 * inf_frac),
            "config": {"workload": "plain Groth16 prover, BN254, synthetic R1CS 2^%d constraints, 1xH100 per replica "
                                   "(BASELINE.json configs[1])" % target_log_m, "arm": "host CPU (oracle/c port of the reference path)"},
            "cpu_baseline": {"value": v, "unit": "proofs/s", "cores": int(cores), "kind": "port", "sample": sample},
            "e2e": {"value": v, "unit": "proofs/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}


def plonk_prove(key, public_inputs, witness, blinders_mont):
    """oracle_plonk_prove: `key` = the dict co_snarks_b200.binding.PlonkKey takes (Montgomery numpy arrays, BN254).
    -> (points [9, 8], evals [6, 4])."""
    from co_snarks_b200.binding import PlonkKeyDesc, u32p, u64p  # type definition only
    d = PlonkKeyDesc()
    keep = []

    def arr(x, dt):
        a = np.ascontiguousarray(x, dtype=dt)
        keep.append(a)
        return a.ctypes.data_as(u64p if dt == np.uint64 else u32p)
    d.curve = 0
    for k in ("n_vars", "n_public", "domain_size", "n_additions", "n_constraints"):
        setattr(d, k, int(key[k]))
    d.k1_mont, d.k2_mont, d.vk_points = arr(key["k1"], np.uint64), arr(key["k2"], np.uint64), arr(key["vk_points"], np.uint64)
    d.additions_ids, d.additions_factors = arr(key["additions_ids"], np.uint32), arr(key["additions_factors"], np.uint64)
    for k in ("map_a", "map_b", "map_c"):
        setattr(d, k, arr(key[k], np.uint32))
    for i in range(5):
        d.q_coeffs[i], d.q_evals[i] = arr(key["q_coeffs"][i], np.uint64), arr(key["q_evals"][i], np.uint64)
    for i in range(3):
        d.s_coeffs[i], d.s_evals[i] = arr(key["s_coeffs"][i], np.uint64), arr(key["s_evals"][i], np.uint64)
    d.lagrange_evals = arr(key["lagrange_evals"], np.uint64)
    pt = np.ascontiguousarray(key["p_tau"], dtype=np.uint64)
    d.p_tau, d.n_p_tau = pt.ctypes.data_as(u64p), pt.shape[0]
    pub = np.ascontiguousarray(public_inputs, dtype=np.uint64)
    wit = np.ascontiguousarray(witness, dtype=np.uint64)
    bl = np.ascontiguousarray(blinders_mont, dtype=np.uint64)
    pts, evs = np.zeros((9, 8), dtype=np.uint64), np.zeros((6, 4), dtype=np.uint64)
    rc = lib().oracle_plonk_prove(C.byref(d), _p(pub), _p(wit), _p(bl), _p(pts), _p(evs))
    assert rc == 0, "oracle_plonk_prove failed (%d)" % rc
    return pts, evs


def time_plonk(key, public_inputs, witness, blinders_mont, reps=1):
    """seconds per Plonk proof of the C restatement (CPU baseline of the Plonk row)."""
    t0 = time.time()
    for _ in range(reps):
        plonk_prove(key, public_inputs, witness, blinders_mont)
    return (time.time() - t0) / reps
