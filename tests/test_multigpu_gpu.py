"""Multi-GPU parity (needs >= 2 CUDA devices; skipped on a 1-GPU machine): a frame-sharded window -- frame <-> pixel
ownership swapped around every motion module through peer memory (fused kernel stores + flag barriers) or through NCCL
all-to-alls -- must reproduce the unsharded engine's latents.  Runs tests/mgpu_worker.py under torchrun."""
import json
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# two runs of the SAME unsharded plan differ by ~1e-3 after a few steps (fp32 atomics reorder sums, fp16 roundings flip
# downstream: tests/test_unet_gpu.py::test_unet_forward_run_to_run_reproducibility); a wrong exchange lands at O(1)
TOL = 5e-3


def _run(world, exchange, port):
    env = dict(os.environ, HALLO_B200_EXCHANGE=exchange, MASTER_ADDR="127.0.0.1", SIZE="32", FRAMES="16")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
                        "--master-addr", "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tests", "mgpu_worker.py")],
                       env=env, capture_output=True, text=True, timeout=900)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("MGPU_RESULT ")]
    assert r.returncode == 0 and lines, r.stdout[-3000:] + r.stderr[-3000:]
    return json.loads(lines[-1][len("MGPU_RESULT "):])


@pytest.mark.parametrize("exchange", ["peer", "nccl"])
def test_frame_sharded_window_matches_unsharded(exchange):
    n = torch.cuda.device_count() if torch.cuda.is_available() else 0
    if n < 2:
        pytest.skip("needs >= 2 CUDA devices")
    world = 2 if n < 4 else (4 if n < 8 else 8)
    res = _run(world, exchange, 29531 if exchange == "peer" else 29532)
    print(res)
    assert all(c == 0 for c in res["device_errors_all_ranks"]), res
    assert res["eager_rel_l2"] < TOL and res["graph_rel_l2"] < TOL, res
