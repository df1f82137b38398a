"""Tensor-parallel generate() with logits processors: every rank returns the same ids, greedy and sampled (needs >= 2
GPUs; `_tp_process_worker.py` under torchrun)."""
import os
import socket
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu


def test_tp_ranks_process_logits_alike():
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    world = 2
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    worker = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_tp_process_worker.py")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
                        "--master-addr", "127.0.0.1", "--master-port", str(port), worker],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert all(f"RANK{i} OK" in r.stdout for i in range(world)), r.stdout[-2000:]
