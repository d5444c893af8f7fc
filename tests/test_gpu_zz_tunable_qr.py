"""CA-CholeskyQR2 on the tunable 2 x 4 x 2 grid: launches tests/mp_worker_tune.py with 16 ranks under torch.distributed.run.

Every rank on cuda:0 runs wherever the GPU tests run (the same peer-layer code, time-sliced; the ranks bootstrap through the host
all-gather because NCCL refuses two ranks on one device).  With 8 GPUs the ranks also run two per GPU."""
import os, subprocess, sys, time
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(per_gpu, timeout=1500):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=16", "--master-addr", "127.0.0.1",
           "--master-port", str(29611 + per_gpu), os.path.join(ROOT, "tests", "mp_worker_tune.py")]
    env = dict(os.environ, CAPITAL_MP_RANKS_PER_GPU=str(per_gpu), CAPITAL_BOOTSTRAP="host")
    t0 = time.time()
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=timeout, env=env)
    assert r.returncode == 0 and "MP_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
    line = [l for l in r.stdout.splitlines() if l.startswith("MP_OK")][0]
    print(f"\n16 ranks, {per_gpu} per GPU, {time.time() - t0:.0f} s: {line}")


def test_tunable_grid_16_ranks_sharing_one_gpu():
    _run(16)


def test_tunable_grid_2_ranks_per_gpu_on_8_gpus():
    if torch.cuda.device_count() < 8:
        pytest.skip("needs 8 GPUs")
    _run(2)
