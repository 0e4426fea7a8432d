#!/bin/bash
# A/B of this tree's library against one built from the parent commit, parent and new alternating (cfg3 three runs
# each, cfg2 / cfg5 / cfg4 two), then bench.py --dump-outputs of both on cfg3, cfg2, cfg5 and cfg4 for an output comparison.
# Usage: bash tools/gpu_ab.sh <parent library .so> [output directory, default: a new temporary directory]
# The new arm also loads its library through SDB_LIB, so that both arms run the same bench.py legs.
PARENT=${1:?parent library}
NEW=sigdigger_b200/libsigdigger_b200.so
O=${2:-$(mktemp -d)}
mkdir -p "$O"; echo "results in $O"
nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv,noheader | tee $O/ab_gpu.txt
run() { # arm, workload, rep
  lib=$PARENT; [ $1 = new ] && lib=$NEW
  out=$O/ab_$2_$1_$3
  SDB_LIB=$lib timeout 300 python bench.py --workload $2 --no-cpu --no-formats --no-single > $out.json 2> $out.err
  python - <<PY
import json
try:
    d = json.load(open("$out.json")); r = d.get("roofline", {})
    print("$2 $1 $3", round(d["value"], 1), round(d["ms_per_step"], 3), r.get("device_ms_per_step", r.get("phases_ms")))
except Exception as ex: print("$2 $1 $3 failed", ex)
PY
}
for w in cfg3:3 cfg2:2 cfg5:2 cfg4:2; do
  for i in $(seq 1 ${w#*:}); do run parent ${w%:*} $i; run new ${w%:*} $i; done
done
for w in cfg3 cfg2 cfg5 cfg4; do
  for arm in parent new; do
    lib=$PARENT; [ $arm = new ] && lib=$NEW
    SDB_LIB=$lib timeout 300 python bench.py --workload $w --steps 2 --warmup 1 --no-cpu --no-formats --no-single \
      --dump-outputs $O/dump_${w}_$arm > /dev/null 2> $O/dump_${w}_$arm.err
  done
  python - <<PY
import glob, os
import numpy as np
a = sorted(glob.glob("$O/dump_${w}_parent/*.npy"))
bad = [os.path.basename(p) for p in a if not np.array_equal(np.load(p), np.load(p.replace("_parent/", "_new/")))]
print("$w outputs:", len(a), "files,", "all equal" if a and not bad else "DIFFER: %s" % bad)
PY
  rm -rf $O/dump_${w}_parent $O/dump_${w}_new
done
