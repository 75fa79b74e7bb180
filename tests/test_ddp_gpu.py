"""Data-parallel parity as pytest (SURVEY.md 8e): two ranks (NCCL on two GPUs, or gloo over CUDA tensors when the box has
one) run tests/ddp_worker.py -- rank-r loss vs the oracle on shard r, rank-averaged gradients vs the mean of the oracle's
shard gradients, Adam moments after a real step, replicas bit-identical afterwards, and one all-reduce of one gradient
buffer per step.  Covers the gradient average (Trainer._average_grads) that eager steps (FactorVAE: BASELINE
configs[3]) and graph replays (configs[1], [4]) share."""
import json
import os
import socket
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


@pytest.mark.parametrize("loss,extra", [("btcvae", []), ("factor", ["--img", "3,64,64", "--per", "32"]),
                                        ("btcvae", ["--img", "3,64,64", "--z", "64", "--per", "24"]),
                                        # SURVEY.md 8f-1: global-batch-exact estimator == ONE process on the whole batch
                                        ("btcvae", ["--img", "3,64,64", "--z", "64", "--per", "24", "--global-btcvae"]),
                                        ("btcvae", ["--per", "40", "--global-btcvae"])])
def test_two_rank_data_parallel_parity(loss, extra):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(_free_port()), os.path.join(ROOT, "tests", "ddp_worker.py"), "--loss", loss] + extra
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    lines = [l for l in r.stdout.splitlines() if l.startswith("DDP_WORKER ")]
    assert lines, r.stdout[-2000:] + "\n" + r.stderr[-6000:]
    rep = json.loads(lines[-1][len("DDP_WORKER "):])
    assert rep["ok"] and r.returncode == 0, json.dumps(rep, indent=1)
    assert rep["world"] == 2
