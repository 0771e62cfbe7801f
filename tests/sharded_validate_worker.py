"""One rank of the sharded trace-check GPU test (tests/test_gpu_sharded_validate.py): `world` processes share GPU 0 and talk
over gloo. argv[1] is a JSON list of cases (tests/sharded_validate_cases.py). Every rank proves its column block with
wf_prove_air_sharded with validation on. A valid trace's proof must equal the proof with validation off and the one-GPU
prover's proof with validation on. A planted violation must refuse the call on every rank with the one-GPU prover's status and
message, write no proof and leave no live device buffer."""
import json
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from sharded_air_worker import opts_of, to_mont  # noqa: E402


def one_gpu(ctx, desc, tr, build, values_fn, nr, nv, opts, mont):
    """(status, message or proof) of the one-GPU prover with validation on."""
    import winterfell_b200 as wf
    full = to_mont(tr) if mont else tr
    ctx.set_validation(1)
    try:
        if build is None:
            return "ok", ctx.prove_air(desc, full, opts, mont=mont)
        return "ok", ctx.prove_air_aux_built(desc, build, full, opts, mont=mont, values_fn=values_fn, num_rands=nr, num_values=nv)
    except wf.WfError as e:
        return "refused", str(e)
    finally:
        ctx.set_validation(0)


def run_case(ctx, comm, case, rank, world):
    import winterfell_b200 as wf
    from sharded_validate_cases import make
    from winterfell_b200 import dist as wd
    log_n = case["log_n"]
    n = 1 << log_n
    desc, tr, build, values_fn, nr, nv = make(case, n, world)
    opts = opts_of(case)
    ctx.set_jit(case.get("jit", 1))
    for k, v in case.get("env", {}).items():
        os.environ[k] = v
    first, count = wd.shard_columns(tr.shape[0], world, rank)
    mode = case.get("trace", "host")
    mont = mode == "mont"
    local = np.ascontiguousarray(tr[first:first + count])
    if mont:
        local = to_mont(local)
    dev = torch.from_numpy(local.view(np.int64)).cuda() if mode == "device" and count else None
    kw = dict(aux_build=build, values_fn=values_fn, num_rands=nr, num_values=nv, mont=mont)

    def prove(stats=None):
        if mode == "device":
            return wd.prove_air_sharded(ctx, comm, desc, None, log_n, opts, device_ptr=dev.data_ptr() if count else 0, local_count=count,
                                        stats=stats, **kw)
        return wd.prove_air_sharded(ctx, comm, desc, local, log_n, opts, stats=stats, **kw)

    want = [one_gpu(ctx, desc, tr, build, values_fn, nr, nv, opts, mont) if rank == 0 else None]
    dist.broadcast_object_list(want, src=0)
    status, want = want[0]
    assert ctx.mem_stats()[0] == 0, "live device buffers before the case"
    on = {}
    ctx.set_validation(1)
    try:
        got = ("ok", prove(on))
    except wf.WfError as e:
        got = ("refused", str(e))
    finally:
        ctx.set_validation(0)
    assert ctx.mem_stats()[0] == 0, "the sharded call left a device buffer live"
    for k in case.get("env", {}):
        os.environ.pop(k)
    if status == "refused":
        assert got == ("refused", want), f"sharded: {got[1] if got[0] == 'refused' else 'a proof'!r}, one GPU: {want!r}"
        return f"refused as one GPU: {want.splitlines()[0]}"
    assert got[0] == "ok", f"sharded prover refused a trace the one-GPU prover accepts: {got[1]!r}"
    off = {}
    proof_off = prove(off)
    assert got[1] == proof_off, "validation changed the sharded proof"
    assert got[1] == want, "sharded proof differs from the one-GPU proof"
    return (f"{len(want)} bytes; collectives {int(off['collectives'])} off, {int(on['collectives'])} on; "
            f"exchanged bytes {int(off['bytes_sent'])} off, {int(on['bytes_sent'])} on")


def main():
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
                msg = run_case(ctx, comm, case, rank, world)
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
