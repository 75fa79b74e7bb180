"""Resuming training on the GPU: a run stopped after 2 epochs and continued in a new process from its saved training
state ends bit-identical to the run that trained 4 epochs without stopping -- parameters, Adam moments and step counts
(FactorVAE's discriminator and its Adam too), the noise and permutation counters and the loss step counter -- and
writes a byte-identical train_losses.log and byte-identical checkpoints.

Every run is a fresh process (tests/resume_worker.py), as after a real preemption, so the continued run's first steps
are its process's first: two eager warm-up steps and the captures, where the uninterrupted run replays graphs.  The
uninterrupted run shares the GPU with the stopped and continued ones, which changes kernel timings but no result.  Every
case anneals across the split (reg_anneal 30, split at step 22), records every 5th step, and ends each epoch on a
short batch (1296 images in batches of 128), so two graph shapes are captured.
"""
import json
import os
import socket
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
WORKER = os.path.join(HERE, "resume_worker.py")


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _start(spec, phase, save_dir, out, eager=False, ranks=1):
    env = dict(os.environ)
    if eager:
        env["DISVAE_CUDA_GRAPH"] = "0"
    cmd = [sys.executable, WORKER, json.dumps(spec), phase, str(save_dir), str(out)]
    if ranks > 1:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(ranks),
               "--master-addr", "127.0.0.1", "--master-port", str(_free_port())] + cmd[1:]
    return phase, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, env=env)


def _wait(run):
    phase, p = run
    try:
        stdout, stderr = p.communicate(timeout=900)
    except subprocess.TimeoutExpired:
        p.kill()
        stdout, stderr = p.communicate()
    assert p.returncode == 0, (phase, stdout[-2000:] + stderr[-6000:])


def _files(d):
    return sorted(f for f in os.listdir(d) if f.startswith("model-") or f == "train_losses.log")


def _assert_same_run(a_dir, b_dir, got, want, what):
    assert got.keys() == want.keys(), what
    for k in want:
        if torch.is_tensor(want[k]):
            assert torch.equal(got[k], want[k]), (what, k)
        else:
            assert got[k] == want[k], (what, k, got[k], want[k])
    assert _files(a_dir) == _files(b_dir), what
    for f in _files(a_dir):
        with open(os.path.join(a_dir, f), "rb") as fa, open(os.path.join(b_dir, f), "rb") as fb:
            assert fa.read() == fb.read(), (what, f)
    with open(os.path.join(a_dir, "train_losses.log")) as f:
        rows = f.read().splitlines()
    assert {r.split(",")[0] for r in rows[1:]} == {"0", "1", "2", "3"}, what      # every epoch recorded


def _split_and_resume(tmp_path, spec, eager=False, ranks=1):
    a, b = tmp_path / "a", tmp_path / "b"
    full = _start(spec, "full", a, tmp_path / "a.pt", eager, ranks)          # runs alongside the stopped run
    try:
        _wait(_start(spec, "first", b, tmp_path / "b1.pt", eager, ranks))
        _wait(_start(spec, "resume", b, tmp_path / "b.pt", eager, ranks))
    finally:
        _wait(full)
    out = []
    for r in range(ranks):
        sub, suffix = ("rank%d" % r, ".rank%d" % r) if ranks > 1 else ("", "")
        want = torch.load(str(tmp_path / "a.pt") + suffix, weights_only=False)
        got = torch.load(str(tmp_path / "b.pt") + suffix, weights_only=False)
        first = torch.load(str(tmp_path / "b1.pt") + suffix, weights_only=False)
        for k, (kind, g, w, f) in enumerate(zip(spec["losses"], got, want, first)):
            d = "m%d_%s" % (k, kind)
            assert f["steps"] == 22 and w["steps"] == 44, (kind, f["steps"], w["steps"])
            assert w["graphs"] == g["graphs"] == (0 if eager else 2), (kind, w["graphs"], g["graphs"])
            _assert_same_run(os.path.join(a, sub, d), os.path.join(b, sub, d), g, w, "%s rank %d" % (kind, r))
        out.append(got)
    return out


@pytest.mark.parametrize("kind,img,loader", [("VAE", 32, "device"), ("betaH", 32, "device"), ("betaB", 64, "device"),
                                             ("btcvae", 32, "host"), ("btcvae", 64, "device"), ("factor", 64, "host"),
                                             ("factor", 32, "device")])
def test_resumed_run_equals_uninterrupted(tmp_path, kind, img, loader):
    _split_and_resume(tmp_path, dict(losses=[kind], img=img, loader=loader, every=1))


def test_resumed_eager_run_equals_uninterrupted(tmp_path):
    _split_and_resume(tmp_path, dict(losses=["factor"], img=32, loader="device", every=1), eager=True)


def test_resumed_sweep_equals_uninterrupted(tmp_path):
    """A two-member sweep stopped and resumed; checkpoints every 3 epochs, so the continued call must number its epochs
    from 2 to write model-3.pt where the uninterrupted one did."""
    got = _split_and_resume(tmp_path, dict(losses=["btcvae", "factor"], img=32, loader="device", every=3, sweep=True))
    assert "perm" in got[0][1]
    for k, kind in enumerate(["btcvae", "factor"]):
        assert _files(tmp_path / "b" / ("m%d_%s" % (k, kind))) == ["model-0.pt", "model-3.pt", "train_losses.log"]
        states = sorted(f for f in os.listdir(tmp_path / "b" / ("m%d_%s" % (k, kind))) if f.startswith("training-state"))
        assert states == ["training-state-0.pt", "training-state-1.pt", "training-state-3.pt"]


def test_resumed_two_rank_run_equals_uninterrupted(tmp_path):
    """Data parallel (two ranks; gloo over CUDA tensors on a one-GPU box): every rank saves and loads its own file and
    ends bit-identical to its own uninterrupted run."""
    _split_and_resume(tmp_path, dict(losses=["btcvae"], img=32, loader="device", every=1), ranks=2)
    for r in range(2):
        assert "training-state-1-rank%d.pt" % r in os.listdir(tmp_path / "b" / ("rank%d" % r) / "m0_btcvae")
