"""The exchange forms at one rank: tests/dist_exchange_check.py under torchrun with a single process.  The script sets up its own
communicator, so at W = 1 it still runs every transport (NCCL send/recv, peer-arena stores, the fenced two-context pipeline, the
split-phase copy-engine form), the general exchange with replicated rows and variable-width columns, and the broadcast.  That reaches
the lane plan, the count matrix, the arena layout and the page assembly of each form on a box with one GPU; tests/test_gpu_dist.py
runs the same script at two ranks."""
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


def _torchrun(script, world, *args, timeout=600):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", str(_free_port()), os.path.join(ROOT, script), *args]
    return subprocess.run(cmd, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=timeout)


def test_one_rank_exchange_and_partitioned_join_match_oracle():
    r = _torchrun("tests/dist_exchange_check.py", 1)
    assert r.returncode == 0, r.stdout[-4000:]
    assert "dist_exchange_check ok" in r.stdout
