"""wf_prove_fib_sharded: one proof over several ranks must be byte-identical to the single-GPU proof (which the other GPU
tests pin to the oracle). The ranks share GPU 0 and use gloo through host staging, so the test runs on a one-GPU box; the
NCCL path is the same library code with device-to-device transfers (bench.py --gpus N, tools/sharded_bench.py)."""
import os
import socket
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(world, k, log_n, ext, hash_id=0, resident=0, fri_min_log=None, extra_env=None):
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    env = dict(os.environ)
    if fri_min_log is not None:
        env["WF_SHARD_FRI_MIN_LOG"] = str(fri_min_log)
    env.update(extra_env or {})
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "tests", "sharded_worker.py"), str(k), str(log_n), str(ext), str(hash_id), str(resident)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=env)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "equal=True" in r.stdout


@pytest.mark.parametrize("world,k,log_n,ext", [(2, 8, 12, 1), (2, 8, 12, 3), (4, 16, 12, 2), (2, 16, 13, 3)])
def test_sharded_proof_equals_single_gpu(world, k, log_n, ext):
    # FRI layers folded on shards down to tiny ranges (WF_SHARD_FRI_MIN_LOG=5): exercises the layer exchange, the per-layer
    # subtree roots and the sharded layer openings
    _run(world, k, log_n, ext, fri_min_log=5)


def test_sharded_proof_default_fri_threshold_and_device_trace():
    # default threshold: at this size every FRI layer is folded after the all-gather; trace block already on the device
    _run(2, 8, 13, 3, resident=1)


def test_sharded_proof_rp64():
    _run(2, 8, 12, 1, hash_id=1, fri_min_log=6)


def test_sharded_proof_with_partitions():
    # ProofOptions::with_partitions(2, 8) (hash_id | 2 << 8 | 8 << 16): the row shards hash column partitions like one GPU does
    _run(2, 8, 12, 3, hash_id=0 | (2 << 8) | (8 << 16), fri_min_log=6)


def test_sharded_proof_communicator_exchange():
    # the trace exchange has two transports: copy-engine pushes into mapped staging buffers (default, the tests above) and the
    # communicator's exchange (WF_PEER_PUSH=0: what a multi-node run would use) — same proof bytes
    env = {"WF_PEER_PUSH": "0"}
    _run(2, 8, 12, 3, fri_min_log=6, extra_env=env)
    _run(4, 16, 13, 1, resident=1, extra_env=env)
