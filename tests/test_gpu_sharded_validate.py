"""wf_prove_air_sharded with validation on (wf_ctx_set_validation): the trace check and the degree check run sharded, each rank
on its share. A valid trace proves to the same bytes as with validation off and as the one-GPU prover; a planted violation
refuses the call on every rank with the one-GPU prover's message, leaves no live buffer, and the next case still proves. The
ranks share GPU 0 over gloo (tests/sharded_validate_worker.py); the cases are those of tests/sharded_validate_cases.py, whose
CPU test shows that each lands on the rank or shard edge it names."""
import json
import os
import socket
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RP64 = 1


def _run(world, cases):
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "tests", "sharded_validate_worker.py"), json.dumps(cases)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1800, env=dict(os.environ))
    out = r.stdout + r.stderr
    assert r.returncode == 0, out[-8000:]
    for q in range(world):
        for i in range(len(cases)):
            assert f"rank {q} case {i} ok" in r.stdout, out[-8000:]
    return r.stdout


def violations(log_n, ext, edges=("0", "edge-1", "edge", "last")):
    """every planted violation, each followed by a valid case, so that every refusal is followed by a proof"""
    ok = {"air": "fib_small_x", "k": 8, "log_n": log_n, "ext": ext}
    out = []
    for at in edges:
        out += [{"plant": "main_transition", "at": at, "log_n": log_n, "ext": ext}, ok]
    for plant in ("assert_last_rank", "asserts_two_ranks", "sequence_two_steps", "exempt_rows", "two_ranks", "aux_init", "aux_term",
                  "aux_dyn_value", "degree_low", "degree_high", "cycled", "periodic_mix"):
        out += [{"plant": plant, "log_n": log_n, "ext": ext}, ok]
    out += [{"plant": "main_and_aux_same_step", "at": "edge-1", "log_n": log_n, "ext": ext},
            {"plant": "aux_degree_straddle", "log_n": log_n, "ext": 3},
            {"air": "perm_rap", "log_n": log_n, "ext": ext}]
    return out


def test_world_2_valid():
    _run(2, [
        {"air": "fib_small_x", "k": 8, "log_n": 11, "ext": 3},
        # 20 columns: a partly filled last segment on rank 1
        {"air": "fib_small_x", "k": 10, "log_n": 11, "ext": 2, "trace": "device"},
        # 2 columns: rank 1 owns none
        {"air": "mulfib2", "log_n": 11, "ext": 2},
        {"air": "sequence_mix", "log_n": 12, "ext": 3, "jit": 0},
        {"air": "rescue_like", "log_n": 11, "ext": 1, "hash": RP64},
        {"air": "perm_rap", "log_n": 11, "ext": 3},
        {"air": "perm_rap", "log_n": 11, "ext": 1, "trace": "mont", "jit": 0},
        {"air": "perm_rap", "dyn": True, "log_n": 12, "ext": 2, "trace": "device"},
        {"air": "fib_small_x", "k": 8, "log_n": 11, "ext": 2, "env": {"WF_PEER_PUSH": "0"}},
        # FibSmall x 16 as a description: 32 columns, one 8-column segment per rank at world 4
        {"air": "fib_small_x", "k": 16, "log_n": 11, "ext": 2},
    ])


def test_world_2_violations():
    _run(2, violations(11, 2))


def test_world_4():
    _run(4, [
        {"air": "fib_small_x", "k": 16, "log_n": 11, "ext": 3, "trace": "device"},
        {"air": "mulfib2", "log_n": 11, "ext": 1, "trace": "mont"},
        {"air": "rescue_like", "log_n": 11, "ext": 2, "jit": 0},
        {"air": "perm_rap", "log_n": 11, "ext": 2, "dyn": True},
        # blowup 2 < world: the aux LDE is extended whole on every rank
        {"air": "perm_rap", "log_n": 12, "ext": 3, "blowup": 2, "queries": 40},
    ] + violations(11, 3))


def test_world_8():
    _run(8, [
        {"air": "fib_small_x", "k": 10, "log_n": 10, "ext": 2},
        {"air": "sequence_mix", "log_n": 10, "ext": 1},
        {"air": "perm_rap", "log_n": 10, "ext": 3, "blowup": 4, "queries": 30},
    ] + violations(10, 1))


def test_larger_trace():
    _run(2, [
        {"air": "fib_small_x", "k": 8, "log_n": 16, "ext": 3},
        {"plant": "main_transition", "at": "edge-1", "log_n": 16, "ext": 3},
        {"air": "perm_rap", "log_n": 16, "ext": 3},
    ])
