"""wf_trace_validate_sharded (winterfell_b200.dist.trace_validate_sharded): on every rank, the report of the whole trace that
the one-GPU wf_trace_validate gives -- its fields, every constraint's first failing step, the expected and actual degrees
and the message -- with check_degrees 0 and 1, for every planted violation and for valid traces, from host, device and
Montgomery main columns and with both ways of passing an aux segment. Refusals are refused on every rank with no live
buffer, and the next case runs. The ranks share GPU 0 over gloo (tests/sharded_trace_validate_worker.py); the cases are
those of tests/sharded_validate_cases.py and tests/sharded_trace_validate_cases.py, whose CPU tests show where each lands."""
import json
import os
import socket
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(world, cases):
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "tests", "sharded_trace_validate_worker.py"), json.dumps(cases)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1800, env=dict(os.environ))
    out = r.stdout + r.stderr
    assert r.returncode == 0, out[-8000:]
    for q in range(world):
        for i in range(len(cases)):
            assert f"rank {q} case {i} ok" in r.stdout, out[-8000:]
    return r.stdout


def planted(log_n, ext, edges=("0", "edge-1", "edge", "last")):
    """every planted violation of both case modules"""
    out = [{"plant": "main_transition", "at": at, "log_n": log_n, "ext": ext} for at in edges]
    for plant in ("assert_last_rank", "asserts_two_ranks", "sequence_two_steps", "exempt_rows", "two_ranks", "aux_init", "aux_term",
                  "aux_dyn_value", "degree_low", "degree_high", "cycled", "periodic_mix",
                  "ranks_first_fail", "last_step_only", "violation_with_degrees"):
        out.append({"plant": plant, "log_n": log_n, "ext": ext})
    out += [{"plant": "main_and_aux_same_step", "at": "edge-1", "log_n": log_n, "ext": ext},
            {"plant": "aux_term", "aux": "cols", "log_n": log_n, "ext": ext},
            {"plant": "aux_degree_straddle", "log_n": log_n, "ext": 3}]
    return out


def valid(log_n, ext):
    return [
        {"air": "fib_small_x", "k": 8, "log_n": log_n, "ext": ext},
        {"air": "fib_small_x", "k": 10, "log_n": log_n, "ext": ext, "trace": "device"},
        {"air": "mulfib2", "log_n": log_n, "ext": ext, "trace": "mont"},
        {"air": "sequence_mix", "log_n": log_n, "ext": ext},
        # 6 columns: one segment, so every rank but rank 0 owns no column
        {"air": "rescue_like", "log_n": log_n, "ext": ext},
        {"air": "perm_rap", "log_n": log_n, "ext": ext},
        {"air": "perm_rap", "log_n": log_n, "ext": ext, "aux": "cols"},
        {"air": "perm_rap", "log_n": log_n, "ext": ext, "aux": "cols", "trace": "mont"},
        {"air": "perm_rap", "log_n": log_n, "ext": ext, "trace": "device"},
        {"air": "linrec", "log_n": log_n, "ext": ext},
        {"air": "rational", "log_n": log_n, "ext": ext, "aux": "cols"},
        {"air": "coupled", "log_n": log_n, "ext": ext},
    ]


def refusals(log_n, ext):
    """each refusal followed by a case that must run"""
    ok = {"air": "fib_small_x", "k": 8, "log_n": log_n, "ext": ext}
    return [{"air": "fib_small_x", "k": 8, "log_n": log_n, "ext": ext, "refuse": "count"}, ok,
            {"air": "fib_small_x", "k": 8, "log_n": 6, "ext": ext, "refuse": "short"}, ok,
            {"air": "perm_rap", "log_n": log_n, "ext": ext, "refuse": "aux_both"}, ok,
            {"air": "fib_small_x", "k": 8, "log_n": log_n, "ext": ext, "refuse": "desc"}, ok]


def test_world_2():
    _run(2, valid(11, 3) + [{"air": "fib_small_x", "k": 16, "log_n": 11, "ext": 2}] + planted(11, 2) + refusals(11, 2))


def test_world_4():
    _run(4, valid(11, 2) + planted(11, 3) + refusals(11, 1))


def test_world_8():
    _run(8, valid(10, 1) + planted(10, 1) + refusals(10, 3))


def test_pool_below_one_context():
    # FibSmall x 16 (32 columns, single segment; FibSmall x 32 needs more registers than the description interpreter has) at
    # 2^17 rows: each rank's pooled bytes at world 4 below one context's. Every process holds a single context, fresh for the call.
    import re
    case = {"air": "fib_small_x", "k": 16, "log_n": 17, "ext": 2, "pool": True}
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "sharded_trace_validate_worker.py"), "--one-gpu", json.dumps(case)],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, (r.stdout + r.stderr)[-4000:]
    one = int(re.search(r"one context pooled bytes (\d+)", r.stdout).group(1))
    out = _run(4, [case])
    per_rank = [int(v) for v in re.findall(r"pooled bytes (\d+)", out)]   # the ranks' lines may share a line of the output
    assert len(per_rank) == 4 and max(per_rank) < one, (per_rank, one)
