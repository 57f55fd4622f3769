"""Rep3CoGroth16::prove INSIDE the library (cs_groth16_rep3_prove): local phase + both network legs in C++.

Mirrors tests/tests/circom/e2e_tests/rep3.rs:36-137 of the reference (all parties return the same proof and
it verifies) and adds byte parity: the masks cancel on opening, so the opened proof must equal the oracle's
plain proof for r = sum r_i.a, s = sum s_i.a.

CPU (not gpu): three party THREADS in one process over in-process mailbox nets (cs_net_peer_connect_local) on
the emulation build; three gloo PROCESSES over the callback transport with OS-entropy states
(cs_rep3_state_create = Rep3State::new's seed exchange); 3 x 2 "GPUs" (main + helper per party).
GPU: the same through real CUDA IPC mailboxes, three processes on the box's GPU(s), and threads on one GPU.
"""
import os
import random
import socket
import sys
import threading

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _shares_for(cv, w, ni, party, seed=5):
    from oracle import groth16 as OG
    wsh = OG.share_rep3(w[ni:], cv.r, random.Random(seed))
    return cv.fr([x for ab in wsh[party] for x in ab]).reshape(-1, 8)


def _check_against_oracle(name, results, curve="bn254"):
    """results: list of (party, A, B, C, rs ints [r.a, r.b, s.a, s.b]) in oracle conventions."""
    from helpers import golden_groth16, ih
    from oracle import groth16 as OG
    from oracle.fields import CURVES
    res = sorted(results)
    proofs = [(a, b, c) for _, a, b, c, _ in res]
    assert proofs[0] == proofs[1] == proofs[2], "parties disagree on the proof"
    z, m, w, g = golden_groth16(name, curve)
    r = CURVES[curve].r
    # replicated randomness is consistent (party i's b == party i-1's a)
    for i in range(3):
        assert res[i][4][1] == res[(i + 2) % 3][4][0] and res[i][4][3] == res[(i + 2) % 3][4][2]
    r_tot = sum(x[4][0] for x in res) % r
    s_tot = sum(x[4][2] for x in res) % r
    assert proofs[0] == OG.prove_plain(z, m, w, r_tot, s_tot), "opened Rep3 proof != plain proof for (sum r, sum s)"
    from kernel_checks import groth16_verifier
    assert groth16_verifier(curve)(OG.vk_from_zkey(z), [ih(x) for x in g["public"]], proofs[0])
    return proofs[0]


def _run_threads(ctx_factory, name, two_gpus=False, curve="bn254"):
    from co_snarks_b200 import binding as B
    from helpers import Conv, golden_groth16, make_key
    cv = Conv(curve)
    z, m, w, g = golden_groth16(name, curve)
    ni = m["num_instance_variables"]
    pub = cv.fr(w[:ni])
    roles = 2 if two_gpus else 1
    ctxs = [[ctx_factory() for _ in range(roles)] for _ in range(3)]
    lib = ctxs[0][0].lib
    pks = [[make_key(c, cv, z, m) for c in row] for row in ctxs]
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
    seeds = [bytes([17 * (i + 1) + k for k in range(32)]) for i in range(3)]
    states = [B.Rep3StateC.from_seeds(lib, i, seeds[i], seeds[(i + 2) % 3]) for i in range(3)]
    out, errs = [], []

    def party(i):
        try:
            sh = _shares_for(cv, w, ni, i)
            A, Bp, Cp, rs = pks[i][0].rep3_prove(nets0[i], nets1[i], states[i], pub, sh,
                                                 pair=pairs[i][0] if two_gpus else None, want_rs=True)
            out.append((i, cv.pt1(A), cv.pt2(Bp), cv.pt1(Cp), cv.fr_back(rs)))
        except Exception as e:  # noqa: BLE001
            errs.append(e)

    th = [threading.Thread(target=party, args=(i,)) for i in range(3)]
    if two_gpus:
        # clone before the mains start consuming their streams
        clones = [states[i].clone() for i in range(3)]

        def helper2(i):
            try:
                pks[i][1].rep3_prove_helper(i, pairs[i][1], clones[i], pub, _shares_for(cv, w, ni, i))
            except Exception as e:  # noqa: BLE001
                errs.append(e)
        th += [threading.Thread(target=helper2, args=(i,)) for i in range(3)]
    for t in th:
        t.start()
    for t in th:
        t.join(timeout=600)
    assert not errs, errs
    sent = [n.bytes_sent for n in nets0 + nets1]
    proof = _check_against_oracle(name, out, curve)
    # the reference exchanges only point-sized messages on this path (four per party)
    assert all(0 < s < 2048 for s in sent)
    for row in pks:
        for pk in row:
            pk.free()
    for n in nets0 + nets1 + ([p for row in pairs for p in row] if pairs else []):
        n.free()
    for s in states:
        s.free()
    return proof


def _emu_factory():
    from co_snarks_b200 import binding as B
    sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
    import build_emu
    emu = build_emu.build()
    return lambda: B.Context(0, lib_path=emu)


def test_rep3_native_three_threads_emu():
    _run_threads(_emu_factory(), "multiplier2")


def test_rep3_native_two_gpus_per_party_emu():
    _run_threads(_emu_factory(), "multiplier2", two_gpus=True)


@pytest.mark.parametrize("name", ["multiplier2", "poseidon"])
def test_rep3_native_three_threads_bls12_381_emu(name):
    """cs_groth16_rep3_prove on BLS12-381 keys: host scalar multiplications on 6-limb Fq, the EC mask and both network
    legs; the opened proof equals the oracle's plain proof and verifies under the BLS12-381 pairing."""
    _run_threads(_emu_factory(), name, curve="bls12_381")


def test_rep3_native_two_gpus_per_party_bls12_381_emu():
    _run_threads(_emu_factory(), "multiplier2", two_gpus=True, curve="bls12_381")


def test_net_mailbox_large_message_emu():
    """cs_net over mailboxes: a message longer than one slot and longer than the credit window arrives intact
    in both directions (chunking + credits)."""
    from co_snarks_b200 import binding as B
    mk = _emu_factory()
    ctxs = [mk() for _ in range(2)]
    nets = [B.Net.peer(ctxs[i], i, 2) for i in range(2)]
    for n in nets:
        n.connect_local(nets)
    rng = random.Random(1)
    msgs = [bytes(rng.randrange(256) for _ in range(20000)), bytes(rng.randrange(256) for _ in range(1025)), b"", b"x"]
    got = [[], []]

    def run(i):
        for mmsg in msgs:
            if i == 0:
                nets[0].send(1, mmsg)
                got[0].append(nets[0].recv(1, len(mmsg)))
            else:
                got[1].append(nets[1].recv(0, len(mmsg)))
                nets[1].send(0, mmsg[::-1])
    th = [threading.Thread(target=run, args=(i,)) for i in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join(timeout=120)
    assert got[1] == msgs and got[0] == [x[::-1] for x in msgs]
    for n in nets:
        n.free()


def test_net_mailbox_sendrecv_ring_emu():
    """cs_net_sendrecv: three parties each send 700 KB to the next and take 700 KB from the previous AT THE SAME TIME;
    that is more than the 8 x 64 KB credit window, so send-then-recv would dead-lock; also the empty message."""
    from co_snarks_b200 import binding as B
    mk = _emu_factory()
    ctxs = [mk() for _ in range(3)]
    nets = [B.Net.peer(ctxs[i], i, 3) for i in range(3)]
    for n in nets:
        n.connect_local(nets)
    msgs = [np.random.default_rng(i).integers(0, 256, 700_000, dtype=np.uint8).tobytes() for i in range(3)]
    got, errs = {}, []

    def run(i):
        try:
            got[i] = nets[i].sendrecv((i + 1) % 3, msgs[i], (i + 2) % 3, len(msgs[i]))
            assert nets[i].sendrecv((i + 2) % 3, b"", (i + 1) % 3, 0) == b""
        except Exception as e:  # noqa: BLE001
            errs.append(e)
    th = [threading.Thread(target=run, args=(i,)) for i in range(3)]
    for t in th:
        t.start()
    for t in th:
        t.join(timeout=120)
    assert not errs, errs
    assert all(got[i] == msgs[(i + 2) % 3] for i in range(3))
    assert all(n.bytes_sent == 700_000 for n in nets)
    for n in nets:
        n.free()


def test_rep3_state_streams_emu():
    """cs_rep3_state: F::rand rejection sampling stays below r; fork derives child seeds from both streams;
    prf() exposes (seed, word position) and rand() advances them."""
    from co_snarks_b200 import binding as B
    from helpers import Conv
    ctx = _emu_factory()()
    lib = ctx.lib
    cv = Conv("bn254")
    s_own, s_prev = bytes(range(32)), bytes(range(32, 64))
    st = B.Rep3StateC.from_seeds(lib, 1, s_own, s_prev)
    peer = B.Rep3StateC.from_seeds(lib, 2, bytes(range(64, 96)), s_own)  # party 2's rng2 is party 1's rng1
    import ctypes as C
    a = np.zeros((2, 4), dtype=np.uint64)
    b = np.zeros((2, 4), dtype=np.uint64)
    for _ in range(20):
        assert lib.cs_rep3_state_rand(st.h, cv.id, B._ptr(a)) == 0
        assert lib.cs_rep3_state_rand(peer.h, cv.id, B._ptr(b)) == 0
        assert B.limbs_to_ints(a)[0] < cv.r and B.limbs_to_ints(a)[1] < cv.r
        assert (a[0] == b[1]).all(), "party i's a must be party i+1's b"
    p = st.prf()
    assert p[0] == s_own and p[2] == s_prev and p[1] >= 160 and p[4] == 12
    h = C.c_void_p()
    assert lib.cs_rep3_state_fork(st.h, C.byref(h)) == 0
    child = B.Rep3StateC(lib, h, 1)
    cp = child.prf()
    assert cp[0] != s_own and cp[1] == 0 and st.prf()[1] == p[1] + 32
    # host ChaCha12 == the device keystream kernel (same block function)
    ks = ctx.chacha_keystream(s_own, 0, 12, 2)
    st2 = B.Rep3StateC.from_seeds(lib, 0, s_own, s_own)
    lib.cs_rep3_state_rand(st2.h, cv.id, B._ptr(a))
    w = np.asarray(ks, dtype=np.uint32).reshape(-1)
    limbs = [int(w[2 * i]) | (int(w[2 * i + 1]) << 32) for i in range(4)]
    limbs[3] &= (1 << 62) - 1
    v = sum(l << (64 * i) for i, l in enumerate(limbs))
    if v < cv.r:
        assert B.limbs_to_ints(a)[0] == v
    for s in (st, peer, child, st2):
        s.free()
    ctx.close()


def _party_proc(rank, port, emu_path, q, name, gpu):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch
    import torch.distributed as dist
    from co_snarks_b200 import binding as B
    from helpers import Conv, golden_groth16, make_key
    dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%d" % port, rank=rank, world_size=3)
    try:
        cv = Conv("bn254")
        z, m, w, g = golden_groth16(name)
        ni = m["num_instance_variables"]
        if gpu:
            ctx = B.Context(rank % torch.cuda.device_count())
            net0, net1 = B.Net.peer(ctx, rank, 3), B.Net.peer(ctx, rank, 3)
            B.connect_peer_nets_over_dist([net0, net1])
        else:
            ctx = B.Context(0, lib_path=emu_path)

            pending = []

            def send(to, data):  # must not block on the receiver (mpc-net queues its sends)
                t = torch.frombuffer(bytearray(data), dtype=torch.uint8)
                pending.append((dist.isend(t, to), t))

            def recv(frm, nbytes):
                t = torch.empty(nbytes, dtype=torch.uint8)
                dist.recv(t, frm)
                return t.numpy().tobytes()
            net0 = B.Net.callbacks(ctx.lib, rank, 3, send, recv)
            net1 = net0
        pk = make_key(ctx, cv, z, m)
        state = B.Rep3StateC.create(net0)  # OS entropy + reshare, as Rep3State::new
        A, Bp, Cp, rs = pk.rep3_prove(net0, net1, state, cv.fr(w[:ni]), _shares_for(cv, w, ni, rank), want_rs=True)
        q.put((rank, cv.pt1(A), cv.pt2(Bp), cv.pt1(Cp), cv.fr_back(rs), net0.bytes_sent))
        if not gpu:
            for wk, _ in pending:
                wk.wait()
        dist.barrier()
        pk.free()
        net0.free()
        if net1 is not net0:
            net1.free()
        state.free()
        ctx.close()
    finally:
        dist.barrier()
        dist.destroy_process_group()


def _run_procs(name, gpu):
    import torch.multiprocessing as mp
    emu = None
    if not gpu:
        sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
        import build_emu
        emu = build_emu.build()
    ctxm = mp.get_context("spawn")
    q = ctxm.Queue()
    port = _free_port()
    procs = [ctxm.Process(target=_party_proc, args=(r, port, emu, q, name, gpu)) for r in range(3)]
    for p in procs:
        p.start()
    res = [q.get(timeout=600) for _ in range(3)]
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    _check_against_oracle(name, [x[:5] for x in res])
    assert all(0 < x[5] < 4096 for x in res)
    # fresh OS entropy: two parties never share a stream they should not (r.a all distinct)
    assert len({x[4][0] for x in res}) == 3


def test_rep3_native_three_processes_callbacks_gloo():
    _run_procs("multiplier2", gpu=False)


@pytest.mark.gpu
def test_rep3_native_three_processes_ipc_mailboxes_gpu():
    """Three party processes on the box's GPU(s) (one shared GPU on a 1-GPU box), CUDA IPC mailboxes."""
    _run_procs("poseidon", gpu=True)


@pytest.mark.gpu
def test_rep3_native_three_threads_gpu():
    from co_snarks_b200 import binding as B
    _run_threads(lambda: B.Context(0), "poseidon")


@pytest.mark.gpu
def test_rep3_native_two_gpus_per_party_threads_gpu():
    from co_snarks_b200 import binding as B
    import torch
    nd = torch.cuda.device_count()
    k = [0]

    def mk():
        k[0] += 1
        return B.Context((k[0] - 1) % nd)
    _run_threads(mk, "poseidon", two_gpus=True)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["multiplier2", "poseidon"])
def test_rep3_native_three_threads_bls12_381_gpu(name):
    from co_snarks_b200 import binding as B
    _run_threads(lambda: B.Context(0), name, curve="bls12_381")


@pytest.mark.gpu
def test_rep3_native_two_gpus_per_party_threads_bls12_381_gpu():
    from co_snarks_b200 import binding as B
    import torch
    nd = torch.cuda.device_count()
    k = [0]

    def mk():
        k[0] += 1
        return B.Context((k[0] - 1) % nd)
    _run_threads(mk, "poseidon", two_gpus=True, curve="bls12_381")
