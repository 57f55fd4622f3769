"""Batched plain Groth16 proofs against the same proofs made one call at a time, on one GPU.

Synthetic keys (workloads/synth_groth16.py; BN254, or BLS12-381 with --curve) at 2^10 .. 2^20; K proofs with random
witnesses (the timing does not depend on whether they satisfy the R1CS).  Per (size, K) one JSON line:
  * batch_proofs_per_s: K / the wall time of one cs_groth16_prove_plain_batch call (host witnesses; the call returns
    after the device has drained), median of the timed calls after a warm-up call;
  * seq_proofs_per_s: the same K proofs by K cs_groth16_prove_plain calls on the same key;
  * batch_cpu_ms_per_proof / seq_cpu_ms_per_proof: process CPU time per proof (this includes the host thread's wait in
    the CUDA runtime's synchronisation, so it is an upper bound on the host work);
  * batch_kernel_ms: device time of one batch call by kernel family (torch.profiler, CUDA activities, a separate call):
    sort (digits, bucket sort, views, slice order), accumulation (k_msm_accum*), reduction (bucket reduction, final sums,
    group combine), point (k_point_*: the single-point work), ntt, witness map (spmv, products), other;
  * identical: every batch proof equals its sequential proof byte for byte.
The first line names the GPU and its power limit.  K * 2^lg is capped at 2^26 (the host witness arrays).

    python tools/time_groth16_batch.py [--sizes 10,12,14,16,18,20] [--ks 1,8,64,256] [--reps 3] [--curve bls12_381]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from co_snarks_b200 import binding as B  # noqa: E402
from workloads.random_groth16 import rand_fr_limbs  # noqa: E402
from workloads.synth_groth16 import SynthGroth16  # noqa: E402

FAMILIES = (("point", ("k_point_",)), ("accumulation", ("k_msm_accum",)),
            ("reduction", ("k_msm_reduce", "k_msm_final_sum", "k_msm_combine")),
            ("sort", ("k_msm_bin", "k_msm_scan", "k_msm_view", "k_msm_slice")), ("ntt", ("k_ntt",)),
            ("witness_map", ("k_spmv", "k_plain_mul_sub")))


def gpu_line():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clk = (x.strip() for x in out.split(","))
    return {"gpu": name, "power_limit": power, "max_sm_clock": clk}


def kernel_ms(fn):
    """device time of fn()'s kernels by family"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
    out = {k: 0.0 for k, _ in FAMILIES}
    out["other"] = 0.0
    for ev in prof.key_averages():
        us = getattr(ev, "device_time_total", None)
        if us is None:
            us = ev.cuda_time_total
        if not us:
            continue
        fam = next((k for k, pre in FAMILIES if any(p in ev.key for p in pre)), "other")
        out[fam] += us / 1e3
    return {k: round(v, 3) for k, v in out.items()}


def timed(fn, reps):
    fn()  # warm-up: scratch grows, modules load
    wall, cpu = [], []
    for _ in range(reps):
        t0, c0 = time.perf_counter(), time.process_time()
        res = fn()
        wall.append(time.perf_counter() - t0)
        cpu.append(time.process_time() - c0)
    return res, statistics.median(wall), statistics.median(cpu)


def run(ctx, pk, lg, ni, nw, K, reps):
    rng = np.random.default_rng(lg * 1000 + K)
    pubs = rand_fr_limbs(rng, K * ni).reshape(K, ni, 4)
    pubs[:, 0] = pubs[0, 0]
    wits = rand_fr_limbs(rng, K * nw).reshape(K, nw, 4)
    rs, ss = rand_fr_limbs(rng, K), rand_fr_limbs(rng, K)

    def batch():
        return pk.prove_plain_batch(pubs, wits, rs, ss)

    def seq():
        out = [pk.prove_plain(pubs[j], wits[j], rs[j:j + 1], ss[j:j + 1]) for j in range(K)]
        return tuple(np.stack([o[i] for o in out]) for i in range(3))

    got, tb, cb = timed(batch, reps)
    exp, ts, cs = timed(seq, reps)
    same = all(np.array_equal(g, e) for g, e in zip(got, exp))
    return {"curve": "bn254" if pk.curve == B.CS_BN254 else "bls12_381", "log_n": lg, "K": K,
            "batch_proofs_per_s": round(K / tb, 1), "seq_proofs_per_s": round(K / ts, 1),
            "speedup": round(ts / tb, 2), "batch_ms": round(tb * 1e3, 2), "seq_ms": round(ts * 1e3, 2),
            "batch_cpu_ms_per_proof": round(cb * 1e3 / K, 3), "seq_cpu_ms_per_proof": round(cs * 1e3 / K, 3),
            "batch_kernel_ms": kernel_ms(batch), "identical": same}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="10,12,14,16,18,20")
    ap.add_argument("--ks", default="1,8,64,256")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--curve", default="bn254", choices=["bn254", "bls12_381"])
    a = ap.parse_args()
    print(json.dumps(gpu_line()), flush=True)
    ctx = B.Context(0)
    ok = True
    for lg in (int(x) for x in a.sizes.split(",")):
        syn = SynthGroth16(ctx, lg, curve=a.curve)
        pk = syn.make_key()
        ni, nw = syn.public_inputs.shape[0], syn.private_witness.shape[0]
        for K in (int(x) for x in a.ks.split(",")):
            if K << lg > 1 << 26:
                print(json.dumps({"log_n": lg, "K": K, "skipped": "K * 2^lg > 2^26"}), flush=True)
                continue
            line = run(ctx, pk, lg, ni, nw, K, a.reps)
            ok = ok and line["identical"]
            print(json.dumps(line), flush=True)
        pk.free()
    ctx.close()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
