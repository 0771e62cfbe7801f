set -x
mkdir -p gpurun_out
run() { # name nproc port env...
  name=$1; np=$2; port=$3; shift 3
  env "$@" timeout 200 python -m torch.distributed.run --nnodes=1 --nproc-per-node $np --master-addr 127.0.0.1 --master-port $port bench.py --gpus $np --steps 4 --warmup 3 --no-cpu-baseline --no-sub-record > gpurun_out/s2_bench_$name.json 2> gpurun_out/s2_bench_$name.err
  tail -3 gpurun_out/s2_bench_$name.err
  python - <<PY
import json
for l in open('gpurun_out/s2_bench_$name.json'):
    if l.startswith('{'):
        d=json.loads(l); print('$name', d['n_gpus'], d['value'], d['e2e']['value'], d['stage_ms'], d['comm'].get('step_ms_by_rank'))
PY
}
run g8_push 8 29571 WF_X=0
