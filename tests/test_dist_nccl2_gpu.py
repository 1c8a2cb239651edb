"""GPU (needs >= 2 devices): N-rank NCCL gradient exchange == 1-rank with N x accumulation over the
same shards (SURVEY.md §8e), eager and inside a captured CUDA graph.  Runs tools/dp_equivalence.py
under torch.distributed.run on 2 ranks; skipped on single-GPU boxes (the driver's round-end GPU
tier) — run on a machine with 2 GPUs."""
import json
import os
import socket
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


@pytest.mark.parametrize("peer", [False, True])
@pytest.mark.parametrize("graph", [False, True])
def test_two_rank_nccl_equals_single_rank_accumulation(graph, peer):
    """peer=True: the exchange runs on the library's NVLink peer-memory kernel (csrc/peer.cu) instead of
    NCCL; with graph=True its kernels are nodes of the step's single CUDA graph."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
           "--master-addr", "127.0.0.1", "--master-port", str(_free_port()),
           os.path.join(ROOT, "tools", "dp_equivalence.py")] + (["--graph"] if graph else []) + \
        (["--peer"] if peer else [])
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-3000:]
    line = [l for l in res.stdout.splitlines() if l.startswith("{")][-1]
    rec = json.loads(line)
    assert rec["ranks_identical"] and rec["rel_err"] < 5e-3, rec


def test_peer_exchange_matches_nccl_bit_for_bit():
    """tools/peer_check.py on 2 ranks: awkward slice sizes, repeated calls, graph replay, fp16 + bf16."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
           "--master-addr", "127.0.0.1", "--master-port", str(_free_port()),
           os.path.join(ROOT, "tools", "peer_check.py"), "--mb", "64"]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-3000:]
    rec = json.loads([l for l in res.stdout.splitlines() if l.startswith("{")][-1])
    assert rec["ok"] and "failures" not in rec, rec
