"""The synchronised batch norm writing the fp8 copies of delayed scaling, on both exchanges: NVLink
peer memory and the NCCL all-reduce.  Every output is the bits of the pass without the copies, a
rank without rows included.  The workers are separate processes with their own NCCL process group
(tests/syncbn_fp8_worker.py); one rank always, two ranks when the box has two GPUs."""
import os
import socket
import subprocess
import sys

import pytest
import torch

pytestmark = [pytest.mark.gpu]
HERE = os.path.dirname(os.path.abspath(__file__))


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _run(world, peer):
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", MASTER_PORT=str(_free_port()),
               MEB200_SYNCBN_PEER=peer)
    worker = os.path.join(HERE, "syncbn_fp8_worker.py")
    if world == 1:
        cmd = [sys.executable, worker]
    else:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1",
               f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
               "--master-port", env["MASTER_PORT"], worker]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=240)
    print(r.stdout[-3000:])
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-2000:])
    assert r.stdout.count("SYNCBN_FP8_OK") == world, r.stdout[-2000:]


@pytest.mark.parametrize("peer", ["1", "0"], ids=["peer", "all_reduce"])
def test_syncbn_fp8_one_rank(cuda, peer):
    _run(1, peer)


@pytest.mark.parametrize("peer", ["1", "0"], ids=["peer", "all_reduce"])
def test_syncbn_fp8_two_ranks(cuda, peer):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    _run(2, peer)
