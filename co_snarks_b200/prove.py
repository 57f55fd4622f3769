"""`python -m co_snarks_b200.prove --zkey circuit.zkey --wtns witness.wtns --out proof.json`

The GPU counterpart of `co-circom generate-proof groth16|plonk` for the plain driver
(co-circom/co-circom/src/bin/co-circom.rs:966-1066): zkey -> device-resident key, wtns -> witness,
Groth16::plain_prove with fresh (r, s) or Plonk::plain_prove with fresh blinders (the protocol is read from
the zkey), proof written in snarkjs' JSON layout (decimal strings, the layout of
test_vectors/{Groth16,Plonk}/bn254/multiplier2/circom.proof) plus public.json.

`python -m co_snarks_b200.prove --zkey circuit.zkey --wtns w0.wtns w1.wtns ... --out proof.json` proves several
witnesses of one Groth16 circuit in one batch (cs_groth16_prove_plain_batch) and writes proof_<i>.json (and, with
--public-out public.json, public_<i>.json) for witness i.

`python -m co_snarks_b200.prove --zkey circuit.zkey --rep3-shares s.0 s.1 s.2 --out proof.json` is
`generate-proof groth16 --protocol REP3` for the three parties of one box, from their share files.
"""
import struct
import argparse
import json
import os
import secrets
import time

import numpy as np

from . import binding as B

# scalar-field moduli and snarkjs curve names, by cs_curve id (the key tells which one applies)
R_MOD = {B.CS_BN254: 21888242871839275222246405745257275088548364400416034343698204186575808495617,
         B.CS_BLS12_381: 52435875175126190479447740508185965837690552500527637822603658699938581184513}
CURVE_NAME = {B.CS_BN254: "bn128", B.CS_BLS12_381: "bls12381"}


def _canon(lib, arr, field, curve=B.CS_BN254):
    nl = B.limbs_of(curve, field)
    out = np.zeros_like(arr)
    fn = lib.cs_fq_from_mont if field == "fq" else lib.cs_fr_from_mont
    fn(curve, B._ptr(np.ascontiguousarray(arr)), B._ptr(out), arr.size // nl)
    return B.limbs_to_ints(out.reshape(-1, nl))


def _rand_fr(curve, k):
    r = R_MOD[curve]
    return B.ints_to_limbs(B.to_mont_ints([secrets.randbelow(r) for _ in range(k)], r, 4), 4)


def proof_json(lib, A, Bp, C, curve=B.CS_BN254):
    a, b, c = _canon(lib, A, "fq", curve), _canon(lib, Bp, "fq", curve), _canon(lib, C, "fq", curve)
    return {"pi_a": [str(a[0]), str(a[1]), "1"],
            "pi_b": [[str(b[0]), str(b[1])], [str(b[2]), str(b[3])], ["1", "0"]],
            "pi_c": [str(c[0]), str(c[1]), "1"], "protocol": "groth16", "curve": CURVE_NAME[curve]}


def zkey_protocol(path):
    """1 = Groth16, 2 = Plonk (section 1 of the snarkjs container)."""
    with open(path, "rb") as f:
        head = f.read(12)
        assert head[:4] == b"zkey", "%s: not a zkey file" % path
        (nsec,) = struct.unpack("<I", head[8:12])
        for _ in range(nsec):
            typ, ln = struct.unpack("<IQ", f.read(12))
            if typ == 1:
                return struct.unpack("<I", f.read(4))[0]
            f.seek(ln, 1)
    raise ValueError("%s: no protocol section" % path)


def plonk_proof_json(lib, pts, evs, curve=B.CS_BN254):
    names = ("A", "B", "C", "Z", "T1", "T2", "T3", "Wxi", "Wxiw")
    out = {}
    for k, P in zip(names, pts):
        c = _canon(lib, P, "fq", curve)
        out[k] = ["0", "1", "0"] if not any(c) else [str(c[0]), str(c[1]), "1"]
    e = _canon(lib, evs, "fr", curve)
    proof = {k: out[k] for k in names[:7]}
    for k, v in zip(("eval_a", "eval_b", "eval_c", "eval_s1", "eval_s2", "eval_zw"), e):
        proof[k] = str(v)
    proof["Wxi"], proof["Wxiw"] = out["Wxi"], out["Wxiw"]
    proof["protocol"], proof["curve"] = "plonk", CURVE_NAME[curve]
    return proof


def prove_rep3_from_share_files(args):
    """`co-circom generate-proof groth16 --protocol REP3` for all three parties on this box
    (co-circom.rs:1005-1050): each party reads its CompressedRep3SharedWitness / Rep3SharedWitness share file
    (cs_rep3_witness_read), holds its own context, device-resident key and OS-seeded correlated streams, and runs
    Rep3CoGroth16::prove inside the library (cs_groth16_rep3_prove) over in-process mailbox nets; the parties are three
    host threads sharing the GPU.  Every party must return the same opened proof.
    This is a one-operator convenience (and the test of the file path): one process holds all three share files, so there
    is no privacy between the parties here; separate operators run one party per process over cs_net (bench.py,
    tests/test_rep3_native.py)."""
    import threading
    ctxs = [B.Context(args.device, lib_path=args.lib) for _ in range(3)]
    lib = ctxs[0].lib
    t0 = time.time()
    pks = [B.Groth16Key.from_zkey(c, args.zkey) for c in ctxs]
    cv = pks[0].curve
    inputs = []
    for i, path in enumerate(args.rep3_shares):
        pub, sh, kind = B.read_rep3_witness(lib, path, cv)
        if pub.shape[0] != pks[i].ni:
            raise SystemExit("%s: %d public inputs, the key expects %d" % (path, pub.shape[0], pks[i].ni))
        inputs.append([np.ascontiguousarray(pub), np.ascontiguousarray(sh), kind])
    kinds = {x[2] for x in inputs}
    if len(kinds) != 1:
        raise SystemExit("the three share files are of different kinds (replicated / additive)")
    nets0 = [B.Net.peer(ctxs[i], i, 3) for i in range(3)]
    nets1 = [B.Net.peer(ctxs[i], i, 3) for i in range(3)]
    for i in range(3):
        nets0[i].connect_local(nets0)
        nets1[i].connect_local(nets1)
    seeds = [B.os_random(lib, 32) for _ in range(3)]  # Rep3State::new: every party's seed, shared with the next party
    states = [B.Rep3StateC.from_seeds(lib, i, seeds[i], seeds[(i + 2) % 3]) for i in range(3)]
    t1 = time.time()
    res, errs = {}, []

    def party(i):
        try:
            sh = inputs[i][1]
            if inputs[i][2] != B.CS_REP3:
                # additive (compressed) shares: one reshare makes them replicated (uncompress_shared_witness,
                # co-circom/src/lib.rs:64-73): share_i = (mine_i, previous party's_i)
                out = np.zeros((sh.shape[0], 8), dtype=np.uint64)
                ctxs[i]._check(lib.cs_rep3_replicate_additive(nets0[i].h, B._ptr(sh), sh.shape[0], B._ptr(out)))
                sh = out
            res[i] = pks[i].rep3_prove(nets0[i], nets1[i], states[i], inputs[i][0], sh)
        except Exception as e:  # noqa: BLE001
            errs.append(e)
    th = [threading.Thread(target=party, args=(i,)) for i in range(3)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    if errs:
        raise errs[0]
    t2 = time.time()
    if not all(all((res[i][k] == res[0][k]).all() for k in range(3)) for i in (1, 2)):
        raise SystemExit("the three parties opened different proofs")
    A, Bp, C = res[0][:3]
    with open(args.out, "w") as f:
        json.dump(proof_json(lib, A, Bp, C, cv), f)
    if args.public_out:
        with open(args.public_out, "w") as f:
            json.dump([str(x) for x in _canon(lib, inputs[0][0][1:], "fr", cv)], f)
    print("keys+shares load %.1f ms, Generate proof took %.1f ms (3 parties, Rep3)" % ((t1 - t0) * 1e3, (t2 - t1) * 1e3))
    for x in states + nets0 + nets1 + pks:
        x.free()
    for c in ctxs:
        c.close()


def _numbered(path, i):
    stem, ext = os.path.splitext(path)
    return "%s_%d%s" % (stem, i, ext)


def prove_groth16_batch(args):
    """One cs_groth16_prove_plain_batch call over the witnesses of args.wtns, fresh (r, s) per proof."""
    ctx = B.Context(args.device, lib_path=args.lib)
    t0 = time.time()
    pk = B.Groth16Key.from_zkey(ctx, args.zkey)
    cv = pk.curve
    wits = [B.read_wtns(ctx.lib, w, cv) for w in args.wtns]
    if any(w.shape != wits[0].shape for w in wits):
        raise SystemExit("the witness files differ in length")
    wit = np.stack(wits)
    t1 = time.time()
    K = len(wits)
    rs = _rand_fr(cv, 2 * K)
    A, Bp, C = pk.prove_plain_batch(wit[:, :pk.ni], wit[:, pk.ni:], rs[:K], rs[K:])
    t2 = time.time()
    for i in range(K):
        with open(_numbered(args.out, i), "w") as f:
            json.dump(proof_json(ctx.lib, A[i], Bp[i], C[i], cv), f)
        if args.public_out:
            with open(_numbered(args.public_out, i), "w") as f:
                json.dump([str(x) for x in _canon(ctx.lib, wit[i, 1:pk.ni], "fr", cv)], f)
    print("key+witness load %.1f ms, Generate %d proofs took %.1f ms (one batch)" % ((t1 - t0) * 1e3, K, (t2 - t1) * 1e3))
    pk.free()
    ctx.close()


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--zkey", required=True)
    ap.add_argument("--wtns", nargs="+", default=None,
                    help="witness file; several (Groth16): one batch, proof_<i>.json per witness")
    ap.add_argument("--rep3-shares", nargs=3, default=None, metavar=("PARTY0", "PARTY1", "PARTY2"),
                    help="Groth16, 3-party Rep3: the three parties' share files (co-circom split-witness output) instead of --wtns")
    ap.add_argument("--out", default="proof.json")
    ap.add_argument("--public-out", default=None)
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--lib", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args(argv)
    if args.rep3_shares:
        if zkey_protocol(args.zkey) != 1:
            raise SystemExit("--rep3-shares: Groth16 keys only")
        return prove_rep3_from_share_files(args)
    if not args.wtns:
        raise SystemExit("give --wtns (plain prover) or --rep3-shares")
    if len(args.wtns) > 1:
        if zkey_protocol(args.zkey) != 1:
            raise SystemExit("several --wtns: Groth16 keys only")
        return prove_groth16_batch(args)
    args.wtns = args.wtns[0]
    ctx = B.Context(args.device, lib_path=args.lib)
    t0 = time.time()
    if zkey_protocol(args.zkey) == 2:
        pk = B.PlonkKey.from_zkey(ctx, args.zkey)  # the curve comes from the zkey
        cv = pk.curve
        wit = B.read_wtns(ctx.lib, args.wtns, cv)  # rejects a witness over another field
        t1 = time.time()
        bl = _rand_fr(cv, 11)
        ni = pk.n_public + 1
        pts, evs = pk.prove_plain(np.ascontiguousarray(wit[:ni]), np.ascontiguousarray(wit[ni:]), bl)
        t2 = time.time()
        with open(args.out, "w") as f:
            json.dump(plonk_proof_json(ctx.lib, pts, evs, cv), f)
        if args.public_out:
            with open(args.public_out, "w") as f:
                json.dump([str(x) for x in _canon(ctx.lib, wit[1:ni], "fr", cv)], f)
        print("key+witness load %.1f ms, Generate proof took %.1f ms" % ((t1 - t0) * 1e3, (t2 - t1) * 1e3))
        pk.free()
        ctx.close()
        return
    pk = B.Groth16Key.from_zkey(ctx, args.zkey)  # the curve comes from the zkey
    cv = pk.curve
    wit = B.read_wtns(ctx.lib, args.wtns, cv)
    t1 = time.time()
    rs = _rand_fr(cv, 2)
    A, Bp, C = pk.prove_plain(np.ascontiguousarray(wit[:pk.ni]), np.ascontiguousarray(wit[pk.ni:]), rs[0:1], rs[1:2])
    t2 = time.time()
    with open(args.out, "w") as f:
        json.dump(proof_json(ctx.lib, A, Bp, C, cv), f)
    if args.public_out:
        with open(args.public_out, "w") as f:
            json.dump([str(x) for x in _canon(ctx.lib, wit[1:pk.ni], "fr", cv)], f)
    print("key+witness load %.1f ms, Generate proof took %.1f ms" % ((t1 - t0) * 1e3, (t2 - t1) * 1e3))
    pk.free()
    ctx.close()


if __name__ == "__main__":
    main()
