"""CholInv on one GPU issues the leading bands of R12 and Rinv12 early, on the deferred streams (capital_b200/csrc/
cholinv_local.cu).  Every output tile keeps its k range and its k order, so the two-stream schedule with bands must give the SAME
BITS as the single-stream schedule (ctx.set_overlap(False): no deferred streams, no bands), and count the same GEMM flops.

The default band threshold (band_min) is exercised in-process.  Child processes (a fresh context reads CAPITAL_BAND_MIN) put bands
on the small nodes too (1024), or turn them off, which shows that the bands really run: they add launches.
    python tests/test_gpu_bands.py small|bench   runs those cases and prints one JSON line (what the child does)"""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def compare(n, bcm, ci, split, host):
    """(R equal, Rinv equal, gemm_flops on, gemm_flops off, kernel launches on) of one factorization with overlap on / off"""
    import torch
    import capital_b200 as cb
    topo = cb.topo.square(1, 0, 1)
    ctx = topo.context()
    A = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
    if host:
        A = cb.matrix(n, n, 1, 1, data=A.data.cpu().pin_memory())
    out = []
    launches = 0
    try:
        for overlap in (True, False):
            ctx.set_overlap(overlap)
            args = cb.cholinv.info(ci, split, bcm, "U")
            cb.cholinv.factor(A, args, topo)  # first call: workspaces and outputs allocated
            ctx.reset_counters()
            cb.cholinv.factor(A, args, topo)
            torch.cuda.synchronize()
            cnt = ctx.counters()
            if overlap:
                launches = cnt.kernel_launches
            out.append((args.R.clone(), args.Rinv.clone(), cnt.gemm_flops))
    finally:
        ctx.set_overlap(True)
    (r0, ri0, f0), (r1, ri1, f1) = out
    res = (torch.equal(r0, r1), torch.equal(ri0, ri1), f0, f1, launches)
    del A, out, r0, ri0, r1, ri1
    torch.cuda.empty_cache()
    return res


DEFAULT_CASES = [(4096, -3), (16384, -5), (12000, -4)]


@pytest.mark.parametrize("host", [False, True], ids=["device", "pinned_host"])
@pytest.mark.parametrize("split", [1, 2])
@pytest.mark.parametrize("ci", [0, 1])
@pytest.mark.parametrize("n,bcm", DEFAULT_CASES)
def test_bands_bit_identical_to_single_stream(n, bcm, ci, split, host):
    r_eq, ri_eq, f_on, f_off, _ = compare(n, bcm, ci, split, host)
    assert r_eq and ri_eq, (r_eq, ri_eq)
    assert f_on == f_off


CHILD_CASES = {"small": [(n, bcm, ci, split, host) for n, bcm in ((4096, -3), (6000, -3)) for ci in (0, 1) for split in (1, 2)
                         for host in (False, True)],
               "bench": [(16384, -5, 0, 1, False)]}


def child(which, band_min):
    env = dict(os.environ)
    env.pop("CAPITAL_BAND_MIN", None)
    if band_min is not None:
        env["CAPITAL_BAND_MIN"] = str(band_min)
    r = subprocess.run([sys.executable, os.path.abspath(__file__), which], capture_output=True, text=True, timeout=600, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    assert len(res) == len(CHILD_CASES[which])
    for c in res:
        assert c["equal"] and c["flops_equal"], c
    return res


@pytest.mark.parametrize("which,band_min", [("small", 1024), ("bench", None)], ids=["small_nodes_1024", "bench_default"])
def test_bands_run_and_stay_bit_identical(which, band_min):
    with_bands, without = child(which, band_min), child(which, 1 << 40)
    for a, b in zip(with_bands, without):
        if a["host"]:  # A streaming in from the host: its R12 products follow the arrival of their columns, no bands
            assert a["launches"] == b["launches"], (a, b)
        else:
            assert a["launches"] > b["launches"], (a, b)


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    out = []
    for n, bcm, ci, split, host in CHILD_CASES[sys.argv[1]]:
        r_eq, ri_eq, f_on, f_off, launches = compare(n, bcm, ci, split, host)
        out.append({"n": n, "ci": ci, "split": split, "host": host, "equal": bool(r_eq and ri_eq), "flops_equal": f_on == f_off,
                    "launches": launches})
    print(json.dumps(out))
