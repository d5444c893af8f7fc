"""The grid schedules at their edges: launches tests/mp_worker_grid_edges.py under torch.distributed.run (what it checks is in its
docstring; the table is in tests/grid_edges_reference.py and its schedule is replayed on the CPU by tests/test_grid_edges_cpu.py).

With 2 / 4 / 8 ranks sharing cuda:0 (gloo bootstrap, as tests/test_gpu_multi.py) the run needs one GPU; the one-GPU-per-rank variants
skip where the GPUs are not there.  On 2 and 4 ranks a second run of the odd sizes with CAPITAL_POISON_WORKSPACE=1 (workspaces filled with NaN
before use) must give the digests of the first: a ragged tile that reads workspace nobody wrote shows up there."""
import functools
import os, re, subprocess, sys
import pytest
import torch

import grid_edges_reference as ge

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@functools.lru_cache(maxsize=None)
def run(nproc, same_device, poison=False):
    """the worker's case lines, by case id"""
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}", "--master-addr", "127.0.0.1",
           "--master-port", str(29911 + nproc), os.path.join(ROOT, "tests", "mp_worker_grid_edges.py")]
    env = {k: v for k, v in os.environ.items() if k not in ge.KNOB_NAMES}
    env.pop("CAPITAL_GRID_EDGES_SIZES", None)
    env.pop("CAPITAL_POISON_WORKSPACE", None)
    if same_device:
        env["CAPITAL_MP_SAME_DEVICE"] = "1"
    if poison:
        env["CAPITAL_POISON_WORKSPACE"] = "1"
        env["CAPITAL_GRID_EDGES_SIZES"] = ",".join(str(n) for n in ge.ODD_SIZES[ge.GRIDS[nproc][1]])
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=2400, env=env)
    assert r.returncode == 0 and "MP_OK" in r.stdout, r.stdout[-6000:] + r.stderr[-3000:]
    line = [l for l in r.stdout.splitlines() if l.startswith("MP_OK")][-1]
    print(line)
    return dict(m.split(":", 1) for m in line[len("MP_OK "):].split(" | "))


def check(nproc, same_device):
    lines = run(nproc, same_device)
    table = [ge.case_id(*c) for c in ge.cases(nproc)]
    assert all(t in lines for t in table), [t for t in table if t not in lines]
    for t in table:  # every case says what it was checked for (the worker's exit code says that it held)
        assert ("bits==default=True" if not t.endswith(" default") else "layers-identical=True") in lines[t], lines[t]
    assert sum("launches=" in v for v in lines.values()) == 4 * len({c[0] for c in ge.cases(nproc)})


@pytest.mark.parametrize("nproc", [2, 4, 8])
def test_edges_with_ranks_sharing_one_gpu(nproc):
    check(nproc, True)


@pytest.mark.parametrize("nproc", [2, 4, 8])
def test_edges_with_one_gpu_per_rank(nproc):
    if torch.cuda.device_count() < nproc:
        pytest.skip(f"needs {nproc} GPUs")
    check(nproc, False)


@pytest.mark.parametrize("nproc", [2, 4])  # not 8: with eight ranks time-slicing one GPU the second run takes minutes
def test_poisoned_workspaces_change_no_bit(nproc):
    lines, poisoned = run(nproc, True), run(nproc, True, poison=True)
    sha = lambda v: re.search(r"sha=(\w+)", v).group(1)
    cases = [ge.case_id(*c) for c in ge.cases(nproc, ge.ODD_SIZES[ge.GRIDS[nproc][1]])]
    assert cases and all(t in poisoned for t in cases)
    assert all(sha(poisoned[t]) == sha(lines[t]) for t in cases), [t for t in cases if sha(poisoned[t]) != sha(lines[t])]
