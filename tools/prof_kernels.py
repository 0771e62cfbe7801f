"""Per-kernel device times of full bench.py-shaped proofs (torch.profiler, CUDA activities), per proof.

    python tools/prof_kernels.py [--config cfg3|cfg2] [--proofs K] [--out FILE.json]

Prints one line per kernel (ms per proof, launches per proof), busiest first, plus the library's stage times from one more
proof with its stage events on. Profile in a run of its own: tracing slows the host, so end-to-end numbers come from bench.py.
"""
import argparse
import json
import os
import re
import subprocess
import sys
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import winterfell_b200 as wf  # noqa: E402

CONFIGS = {"cfg3": (32, 22, 3), "cfg2": (4, 20, 1)}   # bench.py's (pairs, log_n, ext)


def short(name):
    """Kernel name without argument lists: `fri_fold_kernel<3, 2>` stays apart from `fri_fold_kernel<1, 2>`."""
    name = re.sub(r"^void ", "", name)
    depth, out = 0, []
    for ch in name:
        if ch == "(" and depth == 0:
            break
        depth += ch == "<"
        depth -= ch == ">"
        out.append(ch)
    return "".join(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="cfg3", choices=sorted(CONFIGS))
    ap.add_argument("--proofs", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    pairs, log_n, ext = CONFIGS[a.config]
    n = 1 << log_n
    opts = np.array([32, 8, 16, ext, 4, 31, 0, 0, 0], dtype=np.uint32)
    trace, results = wf.build_fib_trace(pairs, n)
    dev = torch.from_numpy(trace.view(np.int64)).cuda()
    stream = torch.cuda.Stream()
    ctx = wf.Context(0, stream.cuda_stream)
    with torch.cuda.stream(stream):
        for _ in range(3):
            ctx.prove_fib_dev(dev.data_ptr(), pairs, log_n, results, opts)
        torch.cuda.synchronize()
        acts = [torch.profiler.ProfilerActivity.CUDA]
        with torch.profiler.profile(activities=acts) as prof:
            for _ in range(a.proofs):
                ctx.prove_fib_dev(dev.data_ptr(), pairs, log_n, results, opts)
            torch.cuda.synchronize()
        ctx.set_profiling(True)
        ctx.prove_fib_dev(dev.data_ptr(), pairs, log_n, results, opts)
        stages = {k: round(v, 4) for k, v in ctx.stage_times()}
        ctx.set_profiling(False)
    tot, cnt = defaultdict(float), defaultdict(int)
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            k = short(e.name)
            tot[k] += e.device_time_total / 1e3
            cnt[k] += 1
    rows = sorted(((k, tot[k] / a.proofs, cnt[k] / a.proofs) for k in tot), key=lambda r: -r[1])
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    rec = {"config": a.config, "proofs": a.proofs, "gpu": smi, "stage_ms": stages,
           "kernels": [{"name": k, "ms": round(ms, 4), "launches": c} for k, ms, c in rows]}
    print(smi)
    for k, ms, c in rows:
        print(f"{ms:9.4f} ms {c:7.1f}  {k}")
    print(json.dumps(stages))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
