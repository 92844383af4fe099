"""Source-view sharding over REAL ranks: one process per GPU, gpm_shard_run with its ncclAllGather exchange behind the C-ABI.
Needs >= 2 visible GPUs (skipped otherwise; `python -m pytest tests -m gpu -k nccl` on a multi-GPU machine).  Rank 0 also runs
the unsharded job and compares bit patterns — the sharded result must be identical (reference semantics: gipuma.cu:742-806)."""
import json
import os
import socket
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port() -> int:
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _gpus() -> int:
    import torch
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


def _torchrun(nproc, script_args, timeout=900):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc), "--master-addr", "127.0.0.1",
           "--master-port", str(_free_port())] + script_args
    p = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=timeout)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-4000:]
    lines = [l for l in p.stdout.splitlines() if l.startswith("{")]
    assert lines, p.stdout[-2000:] + p.stderr[-2000:]
    return json.loads(lines[-1])


@pytest.mark.parametrize("exchange", ["nccl"])             # the only exchange; kept as a parameter so the case ids stay the same
@pytest.mark.parametrize("world,args", [
    (2, ["--config", "4", "--rows", "96", "--cols", "128", "--views", "13", "--iters", "2"]),
    (2, ["--config", "2", "--rows", "352", "--cols", "480", "--views", "7", "--iters", "3"]),
    (2, ["--config", "2", "--rows", "353", "--cols", "481", "--views", "7", "--iters", "2"]),     # odd width, partial tiles
])
def test_view_shard_over_real_ranks_equals_single_gpu(world, args, exchange):
    """One ncclAllGather per exchange stage behind gpm_shard_run."""
    if _gpus() < world:
        pytest.skip("needs %d GPUs" % world)
    out = _torchrun(world, [os.path.join("tools", "run_shard_nccl.py")] + args)
    assert out["world"] == world and out["collectives"] > 0 and out["exchange"] == "nccl"
    assert out["bit_identical_to_single_gpu"] is True


def test_hybrid_two_groups_over_nccl():
    """BASELINE configs[4] layout in miniature: 2 groups x 2-way view shard (4 GPUs), or 2 groups x 1 on 2 GPUs."""
    n = _gpus()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    world, shard = (4, 2) if n >= 4 else (2, 1)
    out = _torchrun(world, [os.path.join("tools", "run_shard_nccl.py"), "--config", "5", "--rows", "96", "--cols", "128", "--views", "9",
                            "--iters", "2", "--hybrid", str(shard), "--refs", "2"])
    assert out["all_groups_bit_identical_to_single_gpu"] is True
