#!/bin/bash
# compute-sanitizer over every kernel of libmppib.so (tools/sanitize_run.py): memcheck (out-of-bounds / misaligned global and shared
# accesses, leaks of device memory), racecheck (shared-memory hazards: the mbarrier ring of K3, the per-rollout slots of K2, the
# staged tiles of the horizon and colored K1 and the SYRK, the elite kernel's sorts and last-CTA merge, the in-place Cholesky and inverse of the horizon K4),
# synccheck (barrier / mbarrier misuse), and memcheck of the 2-GPU peer-memory exchange when two GPUs are visible.
#   bash tools/sanitize.sh [outdir] [all|1gpu|2gpu]     (on the GPU box; writes <outdir>/sanitize_<tool>.log and a summary line per tool)
set -u
OUT=${1:-gpurun_out}
MODE=${2:-all}
mkdir -p "$OUT"
cd "$(dirname "$0")/.."
CS=${COMPUTE_SANITIZER:-/usr/local/cuda/bin/compute-sanitizer}
[ "$MODE" = 2gpu ] || for tool in memcheck racecheck synccheck; do
    extra=""
    [ "$tool" = memcheck ] && extra="--leak-check no"   # (a leak check only lists the blocks torch's caching allocator keeps until exit)
    timeout 1500 "$CS" --tool $tool $extra --print-limit 20 --error-exitcode 3 python tools/sanitize_run.py > "$OUT/sanitize_$tool.log" 2>&1
    echo "$tool: exit $? ; $(grep -E 'ERROR SUMMARY|RACECHECK SUMMARY|LEAK SUMMARY' "$OUT/sanitize_$tool.log" | tr '\n' ' ')"
done
if [ "$MODE" != 1gpu ] && [ "$(python -c 'import torch; print(torch.cuda.device_count())')" -ge 2 ]; then
    timeout 1500 "$CS" --tool memcheck --target-processes all --print-limit 20 --error-exitcode 3 \
        python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29577 tools/sanitize_run.py > "$OUT/sanitize_memcheck_2gpu.log" 2>&1
    echo "memcheck 2-GPU exchange: exit $? ; $(grep -E 'ERROR SUMMARY' "$OUT/sanitize_memcheck_2gpu.log" | sort | uniq -c | tr '\n' ' ')"
fi
