"""Multi-GPU parity: when at least two GPUs are visible, launch
``tools/multi_gpu_check.py`` (one rank per GPU, NCCL rendezvous on 127.0.0.1) on two of them.  It checks
that the row-sharded lookup — local search, libtavec's peer-memory candidate exchange (and the NCCL
form), merge — is bit-identical to the single-GPU lookup and agrees with the oracle, including the
float32 split form, the five-query-chunk batch of BASELINE configs[3] and the exact fallback through
``finish()``.  Skipped on single-GPU machines (the host logic is covered on CPU by test_sharded_gloo.py)."""

from __future__ import annotations

import os
import socket
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_sharded_lookup_is_bit_identical_on_two_gpus():
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tools", "multi_gpu_check.py")]
    proc = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert proc.returncode == 0, proc.stdout[-3000:] + proc.stderr[-3000:]
    assert proc.stdout.count("multi-gpu ok") >= 8, proc.stdout
