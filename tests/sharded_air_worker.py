"""One rank of the sharded AIR proof GPU test (tests/test_gpu_sharded_air.py): `world` processes share GPU 0 and talk over
gloo (TorchComm's host-staged mode). argv[1] is a JSON list of cases; for each, every rank proves its column block with
wf_prove_air_sharded, all ranks must hold the same bytes, and rank 0 checks them against the one-GPU entry point's proof, the
oracle verifier and wf_verify_air_batch. A case with "refuse" expects every rank to get an error and no live device buffer."""
import hashlib
import json
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

P = 0xFFFFFFFF00000001


def air_of(case, n):
    """(description, trace, aux build, values_fn, num_rands, num_values) of a case"""
    import airs
    import aux_builds as ab
    name = case["air"]
    if name == "perm_rap":
        desc, tr, builder = airs.perm_rap(n, dyn_last_q=case.get("dyn", False))
        vf = builder.values_fn if case.get("dyn") else None
        return desc, tr, ab.perm_rap_build(), vf, 2, builder.num_values
    if name == "fib_small_x":
        desc, tr = airs.fib_small_x(case["k"], n)
    elif name == "rescue_like":
        desc, tr = airs.rescue_like(n, case.get("width", 6))
    else:
        desc, tr = getattr(airs, name)(n)
    return desc, tr, None, None, 0, 0


def opts_of(case):
    from oracle import oracle as o
    return o.make_opts(num_queries=case.get("queries", 20), blowup=case.get("blowup", 8), grinding=2, ext=case["ext"],
                       folding=case.get("folding", 4), rem_max_deg=case.get("rem", 7), batch_c=case.get("batch_c", 0),
                       hash_id=case.get("hash", 0), num_partitions=case.get("partitions", 1), hash_rate=case.get("hash_rate", 1))


def to_mont(a):
    return np.array([[(int(v) << 64) % P for v in row] for row in a], dtype=np.uint64)


def run_case(ctx, comm, case, rank, world):
    import winterfell_b200 as wf
    from oracle import oracle as o
    from winterfell_b200 import dist as wd
    log_n = case["log_n"]
    n = 1 << log_n
    desc, tr, build, values_fn, nr, nv = air_of(case, n)
    opts = opts_of(case)
    ctx.set_jit(case.get("jit", 1))
    if "fri_min_log" in case:
        os.environ["WF_SHARD_FRI_MIN_LOG"] = str(case["fri_min_log"])
    else:
        os.environ.pop("WF_SHARD_FRI_MIN_LOG", None)
    refuse = case.get("refuse")
    for k, v in case.get("env", {}).items():
        os.environ[k] = v
    # a world that is not a power of two has no column rule: every rank offers the first column
    first, count = (0, 1) if refuse == "world" else wd.shard_columns(tr.shape[0], world, rank)
    mode = case.get("trace", "host")
    local = np.ascontiguousarray(tr[first:first + count])
    mont = mode == "mont"
    if mont:
        local = to_mont(local)
    if refuse == "count" and rank == world - 1:   # one rank passes a block of the wrong width: every rank must still return
        local = np.ascontiguousarray(tr[:count + 1])
    if refuse == "desc":
        desc = desc.copy()
        desc[2] = 20   # constraint 0 of degree 20: too high for the blowup factor (wf_air_check)
    kw = dict(aux_build=build, values_fn=values_fn, num_rands=nr, num_values=nv, mont=mont)
    stats = {}
    if refuse:
        live0 = ctx.mem_stats()[0]
        try:
            wd.prove_air_sharded(ctx, comm, desc, local, log_n, opts, **kw)
        except wf.WfError as e:
            assert ctx.mem_stats()[0] == live0, "a refused call left a device buffer live"
            return f"refused: {e}"
        raise AssertionError(f"case {case} was not refused")
    if mode == "device":
        dev = torch.from_numpy(local.view(np.int64)).cuda() if count else None
        proof = wd.prove_air_sharded(ctx, comm, desc, None, log_n, opts, device_ptr=dev.data_ptr() if count else 0, local_count=count,
                                     stats=stats, **kw)
    else:
        proof = wd.prove_air_sharded(ctx, comm, desc, local, log_n, opts, stats=stats, **kw)
    digest = torch.frombuffer(bytearray(hashlib.sha256(proof).digest()), dtype=torch.uint8)
    all_d = [torch.empty_like(digest) for _ in range(world)]
    dist.all_gather(all_d, digest)
    assert all(bool((d == all_d[0]).all()) for d in all_d), "ranks hold different proofs"
    if rank == 0:
        full = to_mont(tr) if mont else tr
        if build is None:
            want = ctx.prove_air(desc, full, opts, mont=mont)
        else:
            want = ctx.prove_air_aux_built(desc, build, full, opts, mont=mont, values_fn=values_fn, num_rands=nr, num_values=nv)
        assert proof == want, f"sharded proof ({len(proof)} bytes) differs from the one-GPU proof ({len(want)} bytes)"
        h = int(opts[8]) & 0xFF
        if values_fn is None:
            assert o.verify_air(desc, proof, h) == 0, "oracle verifier rejected the proof"
            vals = None
        else:
            assert o.verify_air_dyn(desc, proof, h, values_fn, nr, nv, case["ext"]) == 0, "oracle verifier rejected the proof"
            vals = lambda _j, rand, values: values_fn(rand, values)
        assert list(ctx.verify_air_batch([desc], [proof], h, aux_values_fn=vals)) == [wf.VERIFY_ACCEPT], "wf_verify_air_batch rejected the proof"
    for k in case.get("env", {}):
        os.environ.pop(k)
    return f"{len(proof)} bytes, sharded FRI layers {int(stats['sharded_fri_layers'])}, peer push {int(stats['peer_push'])}"


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
                if rank == 0:
                    print(f"case {i} ok: {json.dumps(case)}: {msg}", flush=True)
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
