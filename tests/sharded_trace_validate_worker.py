"""One rank of the standalone sharded trace-check GPU test (tests/test_gpu_sharded_trace_validate.py): `world` processes share
GPU 0 and talk over gloo. argv[1] is a JSON list of cases (tests/sharded_trace_validate_cases.py, and through it
tests/sharded_validate_cases.py). For each case every rank checks its column block with wf_trace_validate_sharded, with
check_degrees 0 and 1, and the whole report (fields, first failing steps, degrees, message) must equal what the one-GPU
wf_trace_validate gives for the whole trace. Case keys besides the fixture's: "trace" (host, device or mont main columns),
"aux" (build or cols: how a two-segment AIR's aux segment is passed), "refuse" (every rank must get an error, leave no live
buffer, and the next case runs), "pool" (report the rank's pooled bytes after the call; it must be the only case of its run, in a fresh context).
With "--one-gpu CASE" a single process reports the pooled bytes of one context running wf_trace_validate on the whole trace."""
import json
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from sharded_air_worker import to_mont  # noqa: E402


def inputs(case, world):
    """(description, trace, aux kwargs of trace_validate, ext) of a case"""
    import sharded_trace_validate_cases as T
    from oracle import oracle as O
    n = 1 << case["log_n"]
    ext = case["ext"]
    desc, tr, build, _, nr, _ = T.make(case, n, world)
    kw = {}
    if build is not None:
        rand = O.rand_elems((nr, ext), 9)
        kw["rand"] = rand
        if case.get("aux", "build") == "build":
            kw["aux_build"] = build
        else:
            aux = T.aux_of(case, desc, tr, build, rand)
            kw["aux"] = to_mont(aux.reshape(aux.shape[0], -1)).reshape(aux.shape) if case.get("trace") == "mont" else aux
    return desc, tr, kw, ext


def run_case(ctx, comm, case, rank, world):
    import winterfell_b200 as wf
    from winterfell_b200 import dist as wd
    log_n = case["log_n"]
    desc, tr, kw, ext = inputs(case, world)
    mode = case.get("trace", "host")
    mont = mode == "mont"
    first, count = wd.shard_columns(tr.shape[0], world, rank)
    local = np.ascontiguousarray(tr[first:first + count])
    if mont:
        local = to_mont(local)
    dev = torch.from_numpy(local.view(np.int64)).cuda() if mode == "device" and count else None
    refuse = case.get("refuse")

    def sharded(check_degrees, local_count=None):
        if mode == "device":
            return wd.trace_validate_sharded(ctx, comm, desc, None, log_n, ext=ext, mont=mont, check_degrees=check_degrees,
                                             device_ptr=dev.data_ptr() if count else 0, local_count=local_count, **kw)
        return wd.trace_validate_sharded(ctx, comm, desc, local, log_n, ext=ext, mont=mont, check_degrees=check_degrees,
                                         local_count=local_count, **kw)

    assert ctx.mem_stats()[0] == 0, "live device buffers before the case"
    if refuse:
        if refuse == "count":    # the last rank claims one column more than it owns
            call = lambda: sharded(1, local_count=count + 1 if rank == world - 1 else None)  # noqa: E731
        elif refuse == "short":  # fewer than 64 rows per rank
            call = lambda: sharded(1)  # noqa: E731
        elif refuse == "aux_both":   # a two-segment AIR with both aux_build and aux_cols
            kw["aux"] = inputs(dict(case, aux="cols"), world)[2]["aux"]
            call = lambda: sharded(1)  # noqa: E731
        elif refuse == "desc":   # a truncated description
            desc = desc[:3].copy()
            call = lambda: sharded(1)  # noqa: E731
        else:
            raise ValueError(refuse)
        try:
            call()
        except wf.WfError as e:
            assert ctx.mem_stats()[0] == 0, "a refused call left a device buffer live"
            return f"refused: {str(e).splitlines()[0]}"
        raise AssertionError("the call was not refused")
    full = to_mont(tr) if mont else tr
    out = []
    for cd in (0, 1):
        want = [ctx.trace_validate(desc, full, ext=ext, mont=mont, check_degrees=cd, **kw) if rank == 0 else None]
        dist.broadcast_object_list(want, src=0)
        want = want[0]
        got = sharded(cd)
        assert ctx.mem_stats()[0] == 0, "the sharded call left a device buffer live"
        assert got == want, f"check_degrees={cd}: sharded {got!r}, one GPU {want!r}"
        out.append(f"kind {got['kind']}")
    return "; ".join(out) + f"; {got['msg'].splitlines()[0] if got['msg'] else 'valid'}"


def pooled_bytes(ctx, case, world, rank=0):
    """the context's pooled bytes after one call with check_degrees (wf_trace_validate at world 1): the context is fresh and
    its pool keeps every buffer a call frees, so that is the call's high-water mark of device memory"""
    from winterfell_b200 import dist as wd
    desc, tr, kw, ext = inputs(case, world)
    if world == 1:
        ctx.trace_validate(desc, tr, ext=ext, **kw)
    else:
        first, count = wd.shard_columns(tr.shape[0], world, rank)
        wd.trace_validate_sharded(ctx, wd.TorchComm(torch.cuda.current_stream()), desc, tr[first:first + count], case["log_n"], ext=ext, **kw)
    return ctx.mem_stats()[2]


def main():
    if sys.argv[1] == "--one-gpu":   # one process, one context: wf_trace_validate's pooled bytes for a "pool" case
        import winterfell_b200 as wf
        ctx = wf.Context(0)
        print(f"one context pooled bytes {pooled_bytes(ctx, json.loads(sys.argv[2]), 1)}", flush=True)
        ctx.close()
        return
    cases = json.loads(sys.argv[1])
    dist.init_process_group("gloo")
    rank, world = dist.get_rank(), dist.get_world_size()
    import winterfell_b200 as wf
    from winterfell_b200 import dist as wd
    torch.cuda.set_device(0)
    stream = torch.cuda.Stream()
    ctx = wf.Context(0, stream.cuda_stream)
    comm = wd.TorchComm(stream)
    ok = True
    with torch.cuda.stream(stream):
        for i, case in enumerate(cases):
            try:
                msg = (f"pooled bytes {pooled_bytes(ctx, case, world, rank)}" if case.get("pool")
                       else run_case(ctx, comm, case, rank, world))
                print(f"rank {rank} case {i} ok: {json.dumps(case)}: {msg}", flush=True)
            except Exception as e:  # report and keep the ranks in step: every case ends in an all-gather below
                ok = False
                print(f"rank {rank} case {i} FAILED: {json.dumps(case)}: {e!r}", flush=True)
            flag = torch.tensor([1 if ok else 0])
            flags = [torch.empty_like(flag) for _ in range(world)]
            dist.all_gather(flags, flag)
            if not all(int(f) for f in flags):
                ok = False
                break
    ctx.close()
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
