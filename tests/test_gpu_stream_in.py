"""cholinv::factor on one GPU streams A into its workspace by column chunks, upper triangle only, for device and pinned-host input
alike; it no longer clears the top-level block of Rinv that complete_inv = 0 skips (the packed output writes those zeros itself), and
it does not write the RiT blocks of the right spine that nobody reads then.  None of this touches arithmetic, so:
  - device input, pinned-host input and the single-stream schedule (set_overlap(False)) give the same bits, with every workspace
    poisoned with NaN (a read of W's uncopied lower triangle, of the no-longer-cleared Rinv block or of a skipped RiT block would
    show), and the same bits as the schedule that copied all of A and cleared the block first (tests/golden/stream_in_sha256.json);
  - a factorization after others of different matrices in the same context gives what a fresh context gives;
  - inverse, sygst and solve after a complete_inv = 0 factor give what a fresh context gives from the same factors.
    python tests/test_gpu_stream_in.py cases|sequence|fresh DIR   what the child processes do (one JSON line)"""
import hashlib
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "stream_in_sha256.json")
CASES = [(n, bcm, ci, split) for n, bcm in ((4096, -3), (12000, -4), (16384, -5)) for ci in (0, 1) for split in (1, 2)]


def sha(t):
    return hashlib.sha256(t.cpu().numpy().tobytes()).hexdigest()


def run_cases():
    import torch
    import capital_b200 as cb
    topo = cb.topo.square(1, 0, 1)
    ctx = topo.context()
    out = []
    for n, bcm, ci, split in CASES:
        A = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
        hA = cb.matrix(n, n, 1, 1, data=A.data.cpu().pin_memory())
        res = {}
        for name, M, overlap in (("device", A, True), ("host", hA, True), ("single_stream", A, False)):
            ctx.set_overlap(overlap)
            args = cb.cholinv.info(ci, split, bcm, "U")
            cb.cholinv.factor(M, args, topo)
            torch.cuda.synchronize()
            res[name] = (args.R.to("cuda"), args.Rinv.to("cuda"))
        ctx.set_overlap(True)
        R, Ri = res["device"]
        out.append({"case": [n, bcm, ci, split], "finite": bool(torch.isfinite(R).all() and torch.isfinite(Ri).all()),
                    "equal": {k: bool(torch.equal(R, v[0]) and torch.equal(Ri, v[1])) for k, v in res.items() if k != "device"},
                    "R": sha(R), "Rinv": sha(Ri)})
        del A, hA, res, R, Ri
        torch.cuda.empty_cache()
    return out


def matrices(cb, topo, n):
    A = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
    return A, cb.matrix(n, n, 1, 1, data=A.data * 2.0 + 1.0)  # another SPD matrix: 2 A + 1 1^T


def derived(cb, torch, topo, args, n):
    """hashes of inverse, sygst (itype 1) and solve from the factors in args"""
    _, A1 = matrices(cb, topo, n)
    B = torch.arange(n * 3, dtype=torch.float64, device="cuda").reshape(n, 3).sin()
    return {"inverse": sha(cb.cholinv.inverse(args, topo)), "sygst": sha(cb.cholinv.sygst(A1, args, topo)),
            "solve": sha(cb.cholinv.solve(args, B, topo))}


SEQ_N = ((4096, -3), (12000, -4))


def run_sequence(dirname):
    import torch
    import capital_b200 as cb
    topo = cb.topo.square(1, 0, 1)
    out = []
    for n, bcm in SEQ_N:
        A2, A1 = matrices(cb, topo, n)
        args = cb.cholinv.info(0, 1, bcm, "U")
        cb.cholinv.factor(A2, args, topo)
        first = (sha(args.R), sha(args.Rinv))
        # other matrices and other settings in the same context: a complete inverse fills every workspace block
        for ci, split in ((1, 1), (0, 2), (1, 2)):
            cb.cholinv.factor(A1, cb.cholinv.info(ci, split, bcm, "U"), topo)
        hA2 = cb.matrix(n, n, 1, 1, data=A2.data.cpu().pin_memory())
        hargs = cb.cholinv.info(0, 1, bcm, "U")
        cb.cholinv.factor(hA2, hargs, topo)
        cb.cholinv.factor(A2, args, topo)
        again = (sha(args.R), sha(args.Rinv))
        torch.save({"R": args.R.cpu(), "Rinv": args.Rinv.cpu()}, os.path.join(dirname, f"factors_{n}.pt"))
        out.append({"n": n, "first": first, "again": again, "host": (sha(hargs.R), sha(hargs.Rinv)),
                    "derived": derived(cb, torch, topo, args, n)})
    return out


def run_fresh(dirname):
    import torch
    import capital_b200 as cb
    topo = cb.topo.square(1, 0, 1)
    out = []
    for n, bcm in SEQ_N:
        f = torch.load(os.path.join(dirname, f"factors_{n}.pt"))
        args = cb.cholinv.info(0, 1, bcm, "U")
        args.R, args.Rinv = f["R"].cuda(), f["Rinv"].cuda()
        args.local_dim = args.global_dim = n
        out.append({"n": n, "derived": derived(cb, torch, topo, args, n)})
    return out


def child(*argv):
    env = dict(os.environ, CAPITAL_POISON_WORKSPACE="1")
    r = subprocess.run([sys.executable, os.path.abspath(__file__), *argv], capture_output=True, text=True, timeout=1200, env=env,
                       cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def test_stream_in_bit_identical_poisoned():
    res = child("cases")
    assert len(res) == len(CASES)
    with open(GOLDEN) as f:
        golden = {tuple(g["case"]): g for g in json.load(f)}
    for c in res:
        assert c["finite"], c
        assert all(c["equal"].values()), c
        g = golden[tuple(c["case"])]
        assert (c["R"], c["Rinv"]) == (g["R"], g["Rinv"]), (c, g)


def test_consecutive_factors_and_fresh_context(tmp_path):
    seq = child("sequence", str(tmp_path))
    fresh = child("fresh", str(tmp_path))
    for s, f in zip(seq, fresh):
        assert s["first"] == s["again"] == s["host"], s
        assert s["derived"] == f["derived"], (s, f)


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    which = sys.argv[1]
    res = run_cases() if which == "cases" else run_sequence(sys.argv[2]) if which == "sequence" else run_fresh(sys.argv[2])
    print(json.dumps(res))
