"""The standalone trace check of a trace sharded over the GPUs of a node (wf_trace_validate_sharded), against the one-GPU
wf_trace_validate.

Run under torchrun, one process per GPU, at world 1, 2, 4 and 8:
    torchrun --nproc-per-node=W tools/bench_sharded_validate.py [--log-n 22] [--reps 3] [--out profiles/bench_sharded_trace_validate_h100.jsonl]
Workloads: "fib16" = the FibSmall x 16 description (32 columns, ce blowup 2, 32 transition constraints; FibSmall x 32 needs
more registers than the description interpreter has) and
"perm_rap" = tests/airs.py's two-segment AIR with its aux segment built on the device (tests/aux_builds.py perm_rap_build),
both with the cubic extension and check_degrees on. At world 1 the arm is wf_trace_validate on the whole trace; at world > 1
every rank passes its wf_shard_columns block from host memory. Per workload: ms per call (every rep, median; the max over
ranks of each rep), every rank's pooled device bytes after the calls (each workload runs in a fresh context, and the pool
keeps every buffer a call frees, so that is the rank's high-water mark of device memory), and whether every rank's report
equals the one-GPU report of the whole trace (checked when the one-GPU arm fits). The card's name, power limit and max SM
clock are read in the same run. When there are fewer GPUs than ranks, the ranks share GPU 0 over gloo (host-staged
exchanges): the pool figures hold, the times are marked not comparable. The one-GPU arm is not run at a shape where the
header's scratch formula says it does not fit on the card. One JSON object per workload on stdout, appended to --out by
rank 0."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import winterfell_b200 as wf  # noqa: E402
from bench_sharded_air import fib_workload, perm_rap_workload  # noqa: E402
from winterfell_b200 import dist as wd  # noqa: E402

EXT = 3


def card(device):
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", str(device)],
                         capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
    name, watts, mhz = [s.strip() for s in out.rsplit(",", 2)]
    return {"name": name, "power_limit_w": float(watts), "max_sm_clock_mhz": float(mhz)}


def one_gpu_bytes(desc, n, width, aux_width):
    """wf_trace_validate's device memory by the header's formula: the trace, its coefficients, its LDE at the ce blowup, and
    the degree check's ce x (n_main + n_aux * ext) scratch, twice (three times above 2^22 CE rows); aux segments likewise"""
    from trace_validate_ref import Air
    A = Air(desc)
    ceb = 1 << A.log_ce_blowup()
    ce = n * ceb
    k = len(A.degrees) + len(A.aux_degrees) * EXT
    cols = width + aux_width * EXT
    return 8 * (2 * n * cols + ce * cols + ce * k * (3 if ce > (1 << 22) else 2))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, default=22)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--workloads", default="fib16,perm_rap")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    world = int(os.environ.get("WORLD_SIZE", "1"))
    shared = world > torch.cuda.device_count()
    backend = "gloo" if shared else "nccl"
    dist.init_process_group(backend)
    rank = dist.get_rank()
    device = 0 if shared else int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(device)
    n = 1 << args.log_n
    the_card = card(device)
    total = torch.cuda.get_device_properties(device).total_memory

    def gather(vals):
        t = torch.tensor(vals, dtype=torch.float64, device="cuda" if backend == "nccl" else "cpu")
        out = [torch.empty_like(t) for _ in range(world)]
        dist.all_gather(out, t)
        return [[float(x) for x in g] for g in out]

    for name in args.workloads.split(","):
        desc, tr, build = fib_workload(16, n) if name == "fib16" else perm_rap_workload(n)
        kw = {}
        if build is not None:
            from oracle import oracle as O
            kw = {"rand": O.rand_elems((2, EXT), 9), "aux_build": build}
        aux_width = 0 if build is None else int(build[0])
        fits = one_gpu_bytes(desc, n, tr.shape[0], aux_width) < 0.9 * total
        stream = torch.cuda.Stream()
        ctx = wf.Context(device, stream.cuda_stream)
        comm = wd.TorchComm(stream) if world > 1 else None
        first, count = wd.shard_columns(tr.shape[0], world, rank) if world > 1 else (0, tr.shape[0])
        local = np.ascontiguousarray(tr[first:first + count])

        def call():
            if world == 1:
                return ctx.trace_validate(desc, tr, ext=EXT, **kw)
            return wd.trace_validate_sharded(ctx, comm, desc, local, args.log_n, ext=EXT, **kw)

        rec = {"tool": "bench_sharded_validate", "workload": name, "log_n": args.log_n, "width": int(tr.shape[0]), "ext": EXT,
               "world": world, "arm": "wf_trace_validate" if world == 1 else "wf_trace_validate_sharded",
               "backend": backend if world > 1 else None, "card": the_card}
        if world == 1 and not fits:
            rec.update({"skipped": "the one-GPU scratch formula exceeds the card", "formula_gib": round(one_gpu_bytes(desc, n, tr.shape[0], aux_width) / 2**30, 3)})
        else:
            times = []
            warmup, reps = (0, 1) if shared else (args.warmup, args.reps)
            with torch.cuda.stream(stream):
                for i in range(warmup + reps):
                    torch.cuda.synchronize()
                    dist.barrier()
                    t0 = time.perf_counter()
                    rep = call()
                    torch.cuda.synchronize()
                    if i >= warmup:
                        times.append((time.perf_counter() - t0) * 1e3)
            same = None
            if world > 1 and fits and rank == 0:   # the one-GPU report of the whole trace, untimed, in its own context
                one = wf.Context(device, stream.cuda_stream)
                same = one.trace_validate(desc, tr, ext=EXT, **kw) == rep
                one.close()
            per_rank = gather(times + [ctx.mem_stats()[2]])
            per_rep = [max(g[i] for g in per_rank) for i in range(reps)]
            if shared:   # the ranks share one GPU and exchange through host memory: the time is not the sharded validator's
                rec.update({"ms_median": "not comparable: ranks share one GPU over gloo"})
            else:
                rec.update({"ms_median": round(statistics.median(per_rep), 3), "ms_per_rep": [round(x, 3) for x in per_rep]})
            rec.update({"pooled_gib_per_rank": [round(g[reps] / 2**30, 3) for g in per_rank],
                        "kind": rep["kind"], "same_report_as_one_gpu": same})
        ctx.close()
        if rank == 0:
            print(json.dumps(rec), flush=True)
            if args.out:
                with open(args.out, "a") as f:
                    f.write(json.dumps(rec) + "\n")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
