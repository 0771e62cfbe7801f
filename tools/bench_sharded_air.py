"""One proof of a user-described AIR sharded over the GPUs of a node (wf_prove_air_sharded), against the one-GPU entry points.

Run under torchrun, one process per GPU, at world 1, 2, 4 and 8:
    torchrun --nproc-per-node=W tools/bench_sharded_air.py [--log-n 22] [--reps 5] [--out profiles/sharded_air_h100.jsonl]
Workloads: "fib16" = the FibSmall x 16 description (2^22 x 32 columns, cubic extension, Blake3_256) through the generic
constraint evaluator, and "perm_rap" = tests/airs.py's two-segment AIR with its aux segment built on the device
(tests/aux_builds.py perm_rap_build; 2^22 rows, cubic extension). At world 1 the arm is wf_prove_air / wf_prove_air_aux_built;
at world > 1 every rank passes its wf_shard_columns block from host memory. Per workload: ms per proof (every rep, median;
the max over ranks of each rep), the stage split of one proof on rank 0 (wf_ctx_set_profiling), the communication counters,
and on rank 0 whether the proof bytes equal the one-GPU proof of the whole trace. The card's name and power limit are read in
the same run. One JSON object per workload on stdout, appended to --out by rank 0. --backend gloo runs the same sequence with
host-staged exchanges (several ranks may then share one GPU: a functional rehearsal, not a measurement).
--validation: the validation arm instead. Per workload, ms per proof with wf_ctx_set_validation off and on (reps alternated,
max over ranks, median), whether the proof bytes are the same both ways, and every rank's pooled device bytes after the
proofs with validation off, then after those with it on (the pool keeps every buffer a proof frees, so that is the rank's
high-water mark of device memory)."""
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
import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import airs  # noqa: E402
import aux_builds  # noqa: E402
import winterfell_b200 as wf  # noqa: E402
from winterfell_b200 import dist as wd  # noqa: E402


def card(device):
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", str(device)],
                         capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
    name, watts = [s.strip() for s in out.rsplit(",", 1)]
    return {"name": name, "power_limit_w": float(watts)}


def fib_workload(k, n):
    """FibSmall x k as a description (the rules of airs.fib_small_x), trace from the library's builder"""
    tr, res = wf.build_fib_trace(k, n)
    A = airs.AirBuilder(2 * k)
    A.pub = [int(v) for v in res]
    for j in range(k):
        A.constraint(A.sub(A.nxt(2 * j), A.add(A.cur(2 * j), A.cur(2 * j + 1))), 1)
        A.constraint(A.sub(A.nxt(2 * j + 1), A.add(A.cur(2 * j + 1), A.nxt(2 * j))), 1)
        A.assert_single(2 * j, 0, j + 1)
        A.assert_single(2 * j + 1, 0, j + 1)
        A.assert_single(2 * j + 1, n - 1, int(res[j]))
    return A.build(), np.ascontiguousarray(tr, dtype=np.uint64), None


def perm_rap_workload(n):
    desc, tr, _ = airs.perm_rap(n)
    return desc, tr, aux_builds.perm_rap_build()


def opts(ext):
    # 28 queries, blowup 8, grinding 16, folding 8, remainder degree 31 (BASELINE.json's options)
    return np.array([28, 8, 16, ext, 8, 31, 0, 0, wf.HASH_BLAKE3_256], dtype=np.uint32)


def validation_arm(ctx, prove, args, world, barrier):
    def gather(vals):
        t = torch.tensor(vals, dtype=torch.float64, device="cuda" if dist.get_backend() == "nccl" else "cpu")
        out = [torch.empty_like(t) for _ in range(world)]
        dist.all_gather(out, t)
        return [[float(x) for x in g] for g in out]

    def timed(on):
        ctx.set_validation(on)
        barrier()
        t0 = time.perf_counter()
        proof = prove()
        torch.cuda.synchronize()
        ctx.set_validation(0)
        return (time.perf_counter() - t0) * 1e3, proof

    pooled = []
    for on in (0, 1):   # warm-up; the pool's high-water mark after the proofs without, then with, the checks
        for _ in range(args.warmup):
            _, proof = timed(on)
        pooled.append(ctx.mem_stats()[2])
    ms = {0: [], 1: []}
    proofs = {}
    for _ in range(args.reps):
        for on in (0, 1):
            t, proofs[on] = timed(on)
            ms[on].append(t)
    per_rank = gather([ms[0][i] for i in range(args.reps)] + [ms[1][i] for i in range(args.reps)] + pooled)
    R = args.reps
    off = [max(g[i] for g in per_rank) for i in range(R)]
    on = [max(g[R + i] for g in per_rank) for i in range(R)]
    gib = 1 << 30
    return {"ms_median_off": round(statistics.median(off), 3), "ms_median_on": round(statistics.median(on), 3),
            "ms_per_rep_off": [round(x, 3) for x in off], "ms_per_rep_on": [round(x, 3) for x in on],
            "same_proof_bytes": proofs[0] == proofs[1],
            "pooled_gib_per_rank_off": [round(g[2 * R] / gib, 3) for g in per_rank],
            "pooled_gib_per_rank_on": [round(g[2 * R + 1] / gib, 3) for g in per_rank]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, default=22)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--workloads", default="fib16,perm_rap")
    ap.add_argument("--backend", default="nccl", choices=["nccl", "gloo"])
    ap.add_argument("--out", default=None)
    ap.add_argument("--validation", action="store_true")
    args = ap.parse_args()
    dist.init_process_group(args.backend)
    rank, world = dist.get_rank(), dist.get_world_size()
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    device = local_rank if args.backend == "nccl" else 0
    torch.cuda.set_device(device)
    stream = torch.cuda.Stream()
    ctx = wf.Context(device, stream.cuda_stream)
    comm = wd.TorchComm(stream) if world > 1 else None
    n = 1 << args.log_n
    the_card = card(device)
    for name in args.workloads.split(","):
        desc, tr, build = fib_workload(16, n) if name == "fib16" else perm_rap_workload(n)
        o = opts(3)
        first, count = wd.shard_columns(tr.shape[0], world, rank) if world > 1 else (0, tr.shape[0])
        local = np.ascontiguousarray(tr[first:first + count])
        stats = {}

        def prove():
            if world == 1:
                return ctx.prove_air(desc, tr, o) if build is None else ctx.prove_air_aux_built(desc, build, tr, o)
            return wd.prove_air_sharded(ctx, comm, desc, local, args.log_n, o, aux_build=build, stats=stats)

        def barrier():
            torch.cuda.synchronize()
            dist.barrier()

        if args.validation:
            with torch.cuda.stream(stream):
                rec = validation_arm(ctx, prove, args, world, barrier)
            rec.update({"tool": "bench_sharded_air", "arm": "validation", "workload": name, "log_n": args.log_n, "width": int(tr.shape[0]),
                        "ext": 3, "world": world, "backend": args.backend if world > 1 else None, "card": the_card})
            if rank == 0:
                print(json.dumps(rec), flush=True)
                if args.out:
                    with open(args.out, "a") as f:
                        f.write(json.dumps(rec) + "\n")
            continue
        with torch.cuda.stream(stream):
            for _ in range(args.warmup):
                proof = prove()
            times = []
            for _ in range(args.reps):
                barrier()
                t0 = time.perf_counter()
                proof = prove()
                torch.cuda.synchronize()
                times.append((time.perf_counter() - t0) * 1e3)
            barrier()
            ctx.set_profiling(True)
            prove()
            breakdown = {k: round(v, 3) for k, v in ctx.stage_times()}
            ctx.set_profiling(False)
            identical = None
            if world > 1 and rank == 0:   # the one-GPU proof of the whole trace, untimed
                want = ctx.prove_air(desc, tr, o) if build is None else ctx.prove_air_aux_built(desc, build, tr, o)
                identical = proof == want
        t = torch.tensor(times, dtype=torch.float64)
        gathered = [torch.empty_like(t) for _ in range(world)]
        dist.all_gather(gathered, t)
        per_rep = [max(float(g[i]) for g in gathered) for i in range(args.reps)]
        rec = {"tool": "bench_sharded_air", "workload": name, "log_n": args.log_n, "width": int(tr.shape[0]), "ext": 3, "world": world,
               "backend": args.backend if world > 1 else None,
               "arm": "wf_prove_air_sharded" if world > 1 else ("wf_prove_air" if build is None else "wf_prove_air_aux_built"),
               "ms_median": round(statistics.median(per_rep), 3), "ms_per_rep": [round(x, 3) for x in per_rep],
               "breakdown_rank0": breakdown, "proof_bytes": len(proof), "byte_identical_to_one_gpu": identical,
               "comm": {k: v for k, v in stats.items()}, "card": the_card}
        if rank == 0:
            print(json.dumps(rec), flush=True)
            if args.out:
                with open(args.out, "a") as f:
                    f.write(json.dumps(rec) + "\n")
    ctx.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
