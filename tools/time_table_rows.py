"""What compact MSM tables cost a Groth16 proof on one GPU.

BN254 keys built by workloads/random_groth16.py: at 2^20 with 16, 8, 4 and 1 table rows (k = 1, 2, 4, 16 windows per
row; a row count that no budget reaches, because the scratch of its k outweighs the rows it saves, is reported as such)
and, with 4 rows, a 13-bit window (W = 20, k = 5) to see whether a narrower window pays off once k > 1; at 2^24
with the rows the library picks by itself and with 4 rows.  Per configuration one JSON line: table rows and bytes, the
key creation time (table precomputation included), the proof time with the witness resident in HBM (after a warm-up;
the call returns after the device has drained), and the stage times of the A MSM (cs_msm_stage_ms: digits,
scan + scatter, accumulation, folds, reduction).  The first line names the GPU and its power limit.

    python tools/time_table_rows.py [--sizes 20,24] [--proofs 5]    (2^24 builds a 2^24 key first: minutes)
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from co_snarks_b200 import binding as B  # noqa: E402
from workloads.random_groth16 import forced_key, rand_fr_limbs, random_key  # noqa: E402


def gpu_line():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True, check=True).stdout.strip().splitlines()[0]
    name, power = (x.strip() for x in out.split(","))
    return {"gpu": name, "power_limit": power}


def run(ctx, lg, mats, pts, pub, wit, rows, window_bits, nproofs):
    def make():
        return B.Groth16Key(ctx, B.CS_BN254, mats, pts, window_bits)
    if rows:
        try:
            forced_key(ctx, make, rows).free()  # leaves the budget set: time a clean creation under it
        except AssertionError as e:  # the scratch of that k outweighs the rows it saves: no budget picks it
            ctx.set_table_budget(0)
            return {"log_n": lg, "window_bits": window_bits or 16, "rows_requested": rows, "not_reachable": str(e)}
    t0 = time.perf_counter()
    pk = make()
    key_s = time.perf_counter() - t0
    ctx.set_table_budget(0)
    got_rows, tbytes = pk.table_info()
    d_wit = ctx.to_device(wit)
    r_, s_ = rand_fr_limbs(np.random.default_rng(5), 2)
    r_, s_ = r_[None, :].copy(), s_[None, :].copy()
    for _ in range(2):
        pk.prove_plain_device(pub, d_wit, r_, s_)
    ms = []
    for _ in range(nproofs):
        t0 = time.perf_counter()
        pk.prove_plain_device(pub, d_wit, r_, s_)
        ms.append((time.perf_counter() - t0) * 1e3)
    ctx.msm_profile(True)
    pk.prove_plain_device(pub, d_wit, r_, s_)
    stages = ctx.msm_stage_ms()
    ctx.msm_profile(False)
    ctx.free(d_wit)
    pk.free()
    return {"log_n": lg, "window_bits": window_bits or 16, "rows_requested": rows or "auto", "table_rows": got_rows,
            "table_bytes": tbytes, "key_upload_s": round(key_s, 3), "proof_ms_median": round(float(np.median(ms)), 2),
            "proof_ms": [round(x, 2) for x in ms], "a_msm_stage_ms": [round(x, 3) for x in stages]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="20")
    ap.add_argument("--proofs", type=int, default=5)
    a = ap.parse_args()
    print(json.dumps(gpu_line()), flush=True)
    ctx = B.Context(0)
    plan = {20: [(0, 0), (8, 0), (4, 0), (1, 0), (4, 13)], 24: [(0, 0), (4, 0)]}
    for lg in (int(x) for x in a.sizes.split(",")):
        mats, pts, pub, wit = random_key(ctx, lg)
        for rows, wb in plan[lg]:
            print(json.dumps(run(ctx, lg, mats, pts, pub, wit, rows, wb, a.proofs)), flush=True)
        del mats, pts
    ctx.close()


if __name__ == "__main__":
    main()
