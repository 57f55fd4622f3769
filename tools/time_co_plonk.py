"""Rep3 co-Plonk, three parties on three GPUs of one box (products stored into the next party's GPU over NVLink,
openings over NCCL): wall time per proof, max over ranks, proof checked by the oracle's verifier on rank 0.
launch: python -m torch.distributed.run --nnodes=1 --nproc-per-node 3 --master-addr 127.0.0.1 --master-port 29519 \
        tools/time_co_plonk.py [log_n ...]

python tools/time_co_plonk.py --shamir N T [log_n ...]: no torchrun; on cuda:0, three Rep3 party threads and then N
Shamir(N, T) party threads (cs_plonk_shamir_prove), each over in-process mailbox nets, proofs checked by the oracle's
verifier.  Per size: ms per proof for both, the Shamir split into device pair generation and the rounds, pairs,
bytes sent per party, the device's peak memory during a proof above its level at the proof's start, and what each party's
session holds after its proofs (its own high-water mark, keys and contexts aside); the card's power limit is read in
the same call."""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch
import torch.distributed as dist

from co_snarks_b200 import binding as B
from co_snarks_b200.plonk import DistRep3Comm, Rep3CoPlonk
from co_snarks_b200.rep3 import Rep3Network, Rep3State, random_field_limbs
from workloads.synth_plonk import SynthPlonk

R = 21888242871839275222246405745257275088548364400416034343698204186575808495617


def measure(sizes, reps=None):
    """-> {"world": 3, "2p<lg>": {...}} on rank 0 (None elsewhere); needs torchrun with 3 ranks."""
    rank = int(os.environ["RANK"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    assert dist.get_world_size() == 3
    out = measure_group(None, local, sizes, reps)
    dist.destroy_process_group()
    return out


def measure_group(group, local, sizes, reps=None):
    """The same inside an existing process group: `group` = a 3-rank torch.distributed group (None = the world), called
    by its three members only.  -> results on the group's rank 0, None on the other two.
    The whole party runs inside the library (cs_plonk_rep3_prove): step sequence, transcript and openings in C++ over
    CUDA-IPC mailboxes; first-layer products are stored into the next party's arena by the kernels and the n-sized
    openings read the peers' out-vectors over NVLink.  torch.distributed only carries the IPC handles at start-up
    (CS_CO_PLONK_PY=1 selects the round-1 Python driver with NCCL openings instead)."""
    rank = dist.get_rank(group)
    ctx = B.Context(local)
    use_py = bool(os.environ.get("CS_CO_PLONK_PY"))
    net = Rep3Network(group=group, device="cuda")
    cnet = B.Net.peer(ctx, rank, 3)
    B.connect_peer_nets_over_dist([cnet], group=group, device="cuda")
    state_c = B.Rep3StateC.create(cnet)  # Rep3State::new: OS-entropy seeds exchanged over the net
    out = {"world": 3}

    def gather_handles(ptr):
        h = torch.from_numpy(ctx.ipc_export(ptr).copy()).cuda()
        outs = [torch.empty_like(h) for _ in range(3)]
        dist.all_gather(outs, h, group=group)
        return [o.cpu().numpy() for o in outs]
    for lg in sizes:
        t_setup = time.time()
        syn = SynthPlonk(ctx, lg)  # same seeds on every rank -> same circuit and key
        pk = syn.make_key()
        setup_s = time.time() - t_setup
        npub = syn.n_public
        # replicated sharing of the private witness from a common seed (every rank derives all three shares)
        g = np.random.Generator(np.random.PCG64(7))
        wit = syn.private_witness  # Montgomery limbs [m, 4]
        m = wit.shape[0]
        s0, s1 = random_field_limbs(g, m), random_field_limbs(g, m)
        ints = lambda a: np.array(B.limbs_to_ints(a), dtype=object)
        x, a0, a1 = ints(wit), ints(s0), ints(s1)
        sh = [a0, a1, (x - a0 - a1) % R]
        mine = np.stack([B.ints_to_limbs(list(sh[rank]), 4), B.ints_to_limbs(list(sh[(rank + 2) % 3]), 4)], axis=1)
        reps = reps or int(os.environ.get('CS_CO_PLONK_REPS', '4'))
        ms = []
        mapped = []
        if use_py:
            state = Rep3State(net, seed=5000 + lg)
            prover = Rep3CoPlonk(ctx, pk, rank)
            comm = DistRep3Comm(prover, net, peer=True)
            sess = prover.sess
        else:
            sess = B.PlonkRep3Session(ctx, pk, rank)
            ha, ho = gather_handles(sess.arena), gather_handles(sess.d_out)
            nxt, prv = (rank + 1) % 3, (rank + 2) % 3
            mapped = [ctx.ipc_open(ha[nxt]), ctx.ipc_open(ho[prv]), ctx.ipc_open(ho[nxt])]
            sess.connect(mapped[0])
            sess.connect_io(mapped[1], mapped[2])
        sent0 = cnet.bytes_sent
        for i in range(reps):
            torch.cuda.synchronize()
            dist.barrier(group=group)
            t0 = time.perf_counter()
            if use_py:
                trace = [] if (os.environ.get("CS_CO_PLONK_TRACE") and i == reps - 1) else None
                pts, evs = comm.run(prover.prove(state, syn.public_inputs, mine, syn.key["vk_points"], syn.n), trace)
                if trace and rank == 0:
                    print("trace 2^%d (kind, compute ms, exchange ms): %s" % (lg, trace), file=sys.stderr, flush=True)
            else:
                pts, evs = sess.prove(cnet, state_c, syn.public_inputs, mine)
            t = torch.tensor([(time.perf_counter() - t0) * 1e3], dtype=torch.float64, device="cuda")
            dist.all_reduce(t, op=dist.ReduceOp.MAX, group=group)
            ms.append(float(t.item()))
        ok = None
        if rank == 0:
            from helpers import Conv, plonk_proof_from_device
            from oracle import plonk as OP
            from oracle.fields import BN254
            from oracle.pairing_bn254 import pairing_product_is_one
            proof = plonk_proof_from_device(Conv("bn254"), pts, evs)
            ok = bool(OP.verify(BN254, syn.vk_ints(), proof, syn.full_witness[1:npub + 1], pairing_product_is_one))
        t = sum(ms[1:]) / len(ms[1:])
        sent = (net.bytes_sent if use_py else cnet.bytes_sent - sent0) // reps
        out["2p%d" % lg] = {"ms_per_proof": round(t, 2), "proofs_per_s": round(1e3 / t, 2), "verified": ok,
                            "bytes_sent_per_party": int(sent), "setup_s": round(setup_s, 1),
                            "driver": "co_snarks_b200/plonk.py + NCCL openings" if use_py else "cs_plonk_rep3_prove (C++, in-library)"}
        net.bytes_sent = 0
        if use_py:
            comm.close()
            prover.free()
        else:
            ctx.synchronize()
            dist.barrier(group=group)
            for mp in mapped:
                ctx.ipc_close(mp)
            sess.free()
        pk.free()
    dist.barrier(group=group)
    state_c.free()
    cnet.free()
    ctx.close()
    return out if rank == 0 else None


class _PeakMem:
    """Samples the device's used memory every millisecond in a background thread (all parties share the device)."""

    def __init__(self):
        import threading
        free, total = torch.cuda.mem_get_info(0)
        self.base, self.peak, self.total, self.stop = total - free, 0, total, False
        self.th = threading.Thread(target=self._run)
        self.th.start()

    def _run(self):
        while not self.stop:
            free, _ = torch.cuda.mem_get_info(0)
            self.peak = max(self.peak, self.total - free - self.base)
            time.sleep(0.001)

    def done(self):
        self.stop = True
        self.th.join()
        return self.peak


def _party_threads(fn, n):
    import threading
    errs = []

    def run(p):
        try:
            fn(p)
        except Exception as e:  # noqa: BLE001
            errs.append(e)
    th = [threading.Thread(target=run, args=(p,)) for p in range(n)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    if errs:
        raise errs[0]


def measure_threads(sizes, num_parties, threshold, reps=None):
    """Rep3 and Shamir(num_parties, threshold) co-Plonk, every party a thread on cuda:0 -> {"2p<lg>": {...}}."""
    import random
    from helpers import Conv, plonk_proof_from_device
    from oracle import plonk as OP
    from oracle.fields import BN254
    from oracle.pairing_bn254 import pairing_product_is_one
    reps = reps or int(os.environ.get("CS_CO_PLONK_REPS", "3"))
    cv = Conv("bn254")
    import subprocess
    power = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True).stdout.strip()  # read-only query, part of the numbers
    out = {"gpu": torch.cuda.get_device_name(0), "power_limit_w": power, "shamir": [num_parties, threshold]}
    for lg in sizes:
        ctx0 = B.Context(0)
        t_setup = time.time()
        syn = SynthPlonk(ctx0, lg)
        setup_s = time.time() - t_setup
        ctx0.close()
        npub, wit = syn.n_public, syn.full_witness[syn.n_public + 1:]
        rng = random.Random(lg)
        row = {"setup_s": round(setup_s, 1)}
        # ---- Rep3: three threads, products stored straight into the next party's arena (same-process pointers)
        s0 = [rng.randrange(R) for _ in wit]
        s1 = [rng.randrange(R) for _ in wit]
        sh = [s0, s1, [(x - a - b) % R for x, a, b in zip(wit, s0, s1)]]
        mine = [np.stack([cv.fr(sh[p]), cv.fr(sh[(p + 2) % 3])], axis=1) for p in range(3)]
        ctxs = [B.Context(0) for _ in range(3)]
        pks = [B.PlonkKey(c, B.CS_BN254, syn.key) for c in ctxs]
        sess = [B.PlonkRep3Session(ctxs[p], pks[p], p) for p in range(3)]
        nets = [B.Net.peer(ctxs[p], p, 3) for p in range(3)]
        for x in nets:
            x.connect_local(nets)
        for p in range(3):
            sess[p].connect(sess[(p + 1) % 3].arena)
            sess[p].connect_io(sess[(p + 2) % 3].d_out, sess[(p + 1) % 3].d_out)
        seeds = [bytes((31 * p + i) & 0xff for i in range(32)) for p in range(3)]
        states = [B.Rep3StateC.from_seeds(ctxs[0].lib, p, seeds[p], seeds[(p + 2) % 3]) for p in range(3)]
        ms, res = [], {}
        for i in range(reps):
            sent0 = [x.bytes_sent for x in nets]
            t0 = time.perf_counter()
            _party_threads(lambda p: res.__setitem__(p, sess[p].prove(nets[p], states[p], syn.public_inputs, mine[p])), 3)
            ms.append((time.perf_counter() - t0) * 1e3)
        proof = plonk_proof_from_device(cv, *res[0])
        row["rep3"] = {"ms_per_proof": round(min(ms[1:] or ms), 1), "all_ms": [round(x, 1) for x in ms],
                       "verified": bool(OP.verify(BN254, syn.vk_ints(), proof, syn.full_witness[1:npub + 1], pairing_product_is_one)),
                       "bytes_sent_per_party": max(x.bytes_sent - s for x, s in zip(nets, sent0))}
        for x in sess + pks + nets + states:
            x.free()
        for c in ctxs:
            c.close()
        # ---- Shamir(n, t): degree-t shares of the witness
        n, t = num_parties, threshold
        co = [[rng.randrange(R) for _ in wit] for _ in range(t)]
        shares = []
        for p in range(n):
            x = p + 1
            shares.append(cv.fr([(v + sum(c[j] * pow(x, k + 1, R) for k, c in enumerate(co))) % R for j, v in enumerate(wit)]))
        ctxs = [B.Context(0) for _ in range(n)]
        pks = [B.PlonkKey(c, B.CS_BN254, syn.key) for c in ctxs]
        sess = [B.PlonkShamirSession(ctxs[p], pks[p], n, t, p) for p in range(n)]
        nets = [B.Net.peer(ctxs[p], p, n) for p in range(n)]
        for x in nets:
            x.connect_local(nets)
        ms, pair_ms, res, peak = [], [], {}, 0
        for i in range(reps):
            sent0 = [x.bytes_sent for x in nets]
            mon = _PeakMem()
            t0 = time.perf_counter()
            _party_threads(lambda p: res.__setitem__(p, sess[p].prove(nets[p], syn.public_inputs, shares[p])), n)
            ms.append((time.perf_counter() - t0) * 1e3)
            peak = max(peak, mon.done())
            pair_ms.append(max(s.pair_ms() for s in sess))
        proof = plonk_proof_from_device(cv, *res[0][:2])
        k = ms.index(min(ms[1:] or ms))
        row["shamir"] = {"ms_per_proof": round(ms[k], 1), "pair_generation_ms": round(pair_ms[k], 1),
                         "rounds_ms": round(ms[k] - pair_ms[k], 1), "all_ms": [round(x, 1) for x in ms],
                         "verified": bool(OP.verify(BN254, syn.vk_ints(), proof, syn.full_witness[1:npub + 1], pairing_product_is_one)),
                         "pairs": sess[0].pairs(), "pairs_formula_58n_13": 58 * syn.n + 13,
                         "bytes_sent_per_party": [x.bytes_sent - s for x, s in zip(nets, sent0)],
                         "peak_device_bytes_all_parties": int(peak),
                         "session_device_bytes_per_party": [x.device_bytes() for x in sess]}
        for x in sess + pks + nets:
            x.free()
        for c in ctxs:
            c.close()
        out["2p%d" % lg] = row
        print(json.dumps({"2p%d" % lg: row}), file=sys.stderr, flush=True)
    return out


if __name__ == "__main__":
    if len(sys.argv) > 3 and sys.argv[1] == "--shamir":
        print(json.dumps(measure_threads([int(a) for a in sys.argv[4:]] or [20], int(sys.argv[2]), int(sys.argv[3]))))
        sys.exit(0)
    res = measure([int(a) for a in sys.argv[1:]] or [16, 18])
    if res is not None:
        print(json.dumps(res))
