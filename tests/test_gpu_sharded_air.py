"""wf_prove_air_sharded: one proof of a user-described AIR over several ranks must be byte-identical on every rank and to the
one-GPU entry point's proof (wf_prove_air, or wf_prove_air_aux_built for two-segment AIRs), and be accepted by the oracle
verifier and wf_verify_air_batch. The ranks share GPU 0 over gloo (tests/sharded_air_worker.py); each test is one launch of
`world` ranks running a list of cases, so that the process start-up is paid once per world size."""
import json
import os
import socket
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BLAKE3, RP64 = 0, 1


def _run(world, cases):
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "tests", "sharded_air_worker.py"), json.dumps(cases)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1200, env=dict(os.environ))
    out = r.stdout + r.stderr
    assert r.returncode == 0, out[-6000:]
    for i in range(len(cases)):
        assert f"case {i} ok" in r.stdout, out[-6000:]
    return r.stdout


def test_world_2():
    _run(2, [
        # the FibSmall x 8 shape as a description, FRI layers folded on shards
        {"air": "fib_small_x", "k": 8, "log_n": 12, "ext": 3, "fri_min_log": 5},
        # 2 columns: rank 1 owns none
        {"air": "mulfib2", "log_n": 11, "ext": 2},
        {"air": "periodic_mix", "log_n": 11, "ext": 1, "hash": RP64, "jit": 0},
        # sequence tables read at global CE rows; column partitions
        {"air": "sequence_mix", "log_n": 12, "ext": 3, "partitions": 2, "hash_rate": 8, "fri_min_log": 6},
        {"air": "rescue_like", "log_n": 11, "ext": 2},
        {"air": "rescue_like", "log_n": 11, "ext": 1, "jit": 0, "trace": "device"},
        # two-segment AIR, aux segment built on the device: host, device and Montgomery traces
        {"air": "perm_rap", "log_n": 12, "ext": 3, "fri_min_log": 5},
        {"air": "perm_rap", "log_n": 11, "ext": 1, "hash": RP64, "trace": "device", "jit": 0},
        {"air": "perm_rap", "log_n": 11, "ext": 2, "trace": "mont", "env": {"WF_PEER_PUSH": "0"}},
        # an aux assertion whose value depends on the random elements (callback)
        {"air": "perm_rap", "dyn": True, "log_n": 12, "ext": 3, "folding": 8, "rem": 15, "queries": 24},
        # 20 columns: a partly filled last segment on rank 1
        {"air": "fib_small_x", "k": 10, "log_n": 11, "ext": 3, "trace": "device"},
        {"air": "fib_small_x", "k": 10, "log_n": 11, "ext": 2, "env": {"WF_PEER_PUSH": "0"}},
    ])


def test_world_4():
    _run(4, [
        # 6 columns over 4 ranks: three ranks own none
        {"air": "fib_small_x", "k": 3, "log_n": 11, "ext": 2, "trace": "mont"},
        {"air": "fib_small_x", "k": 16, "log_n": 11, "ext": 2, "hash": RP64, "partitions": 2, "hash_rate": 8, "fri_min_log": 5},
        {"air": "sequence_mix", "log_n": 12, "ext": 1, "trace": "device", "env": {"WF_PEER_PUSH": "0"}},
        {"air": "periodic_mix", "log_n": 11, "ext": 3, "jit": 0, "fri_min_log": 5},
        {"air": "rescue_like", "log_n": 11, "ext": 3},
        {"air": "perm_rap", "log_n": 11, "ext": 2, "fri_min_log": 5},
        # blowup 2 < world: the composition and aux LDEs are extended whole on every rank (no coset sharding)
        {"air": "perm_rap", "log_n": 12, "ext": 3, "blowup": 2, "queries": 40, "trace": "device"},
        {"air": "mulfib2", "log_n": 12, "ext": 1, "blowup": 2, "queries": 40},
    ])


def test_world_8():
    _run(8, [
        {"air": "fib_small_x", "k": 4, "log_n": 10, "ext": 2},
        {"air": "perm_rap", "log_n": 10, "ext": 2, "blowup": 4, "queries": 30},
        {"air": "perm_rap", "log_n": 10, "ext": 3, "dyn": True},
        {"air": "mulfib2", "log_n": 10, "ext": 3, "jit": 0},
    ])


def test_refusals_return_on_every_rank():
    # each refused call returns an error on every rank (none is left waiting in a collective) and leaves no buffer live
    _run(2, [
        {"air": "mulfib2", "log_n": 11, "ext": 2, "refuse": "desc"},
        {"air": "fib_small_x", "k": 8, "log_n": 6, "ext": 2, "refuse": "short"},
        {"air": "fib_small_x", "k": 8, "log_n": 11, "ext": 2, "refuse": "count"},
        {"air": "perm_rap", "log_n": 11, "ext": 2, "refuse": "count"},
        # and the ranks still prove after the refusals
        {"air": "perm_rap", "log_n": 11, "ext": 2},
    ])
    _run(3, [{"air": "mulfib2", "log_n": 11, "ext": 2, "refuse": "world"}])
