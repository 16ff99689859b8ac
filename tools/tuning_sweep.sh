#!/bin/bash
# Re-tuning sweep on the GPU at hand, from the repository root after build():
#   1. config 2 (bench.py, headline leg only) with the library defaults (three times: the spread) and under each
#      run-time hook;
#   2. VoxelDownSample, dense-grid path vs hash path (CPHB_VOXEL_NO_DENSE), at grids below and above the L2 size;
#   3. device-to-device copy bandwidth (what roofline.frac should be read against).
# One line per setting on stdout; the bench lines are kept in OUTDIR.
#   tools/tuning_sweep.sh [OUTDIR]
set -u
OUT=${1:-tuning_out}
mkdir -p "$OUT"
nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv,noheader

run() {  # label [VAR=value ...]
    local label=$1; shift
    if env "$@" python bench.py --gpus 1 --steps 10 --warmup 3 --no-extras --no-cpu --no-host-call \
            > "$OUT/$label.json" 2> "$OUT/$label.err"; then
        python -c "import json, sys; d = json.load(open(sys.argv[1]))
print('%-26s value %6.0f it/s  loop %6.0f it/s  T[0][3] %.7f' % (sys.argv[2], d['value'], d['loop']['iters_per_sec'], d['final']['T'][0][3]))" \
            "$OUT/$label.json" "$label"
    else
        echo "$label failed: $(tail -1 "$OUT/$label.err")"
    fi
}

for i in 1 2 3; do run default_$i; done
for v in 2 8; do run cert_gain_$v CPHB_CERT_GAIN=$v; done
run static_sched_0 CPHB_STATIC_SCHED=0

python - <<'EOF'
import os, time
import numpy as np
import cupoch_b200 as cph
from cupoch_b200.testing import datagen

def t_ms(pc, v, reps=10):
    pc.voxel_down_sample(v)
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        d = pc.voxel_down_sample(v)   # returns after the voxel count is read back: a device synchronise
        ts.append(1e3 * (time.perf_counter() - t0))
    return float(np.median(ts)), len(d)

for n, v in ((10_000_000, 0.03), (10_000_000, 0.02), (10_000_000, 0.016), (2_000_000, 0.02)):
    pc = cph.geometry.PointCloud(datagen.uniform_cube(n, 21, hi=(4, 4, 1)))
    cells = int(np.prod(np.ceil(np.array([4, 4, 1]) / v)))
    os.environ.pop("CPHB_VOXEL_NO_DENSE", None)
    dense, m = t_ms(pc, v)
    os.environ["CPHB_VOXEL_NO_DENSE"] = "1"
    hashed, _ = t_ms(pc, v)
    os.environ.pop("CPHB_VOXEL_NO_DENSE")
    print("voxel n=%d v=%g cells~%d (dense accumulators %.0f MB) voxels=%d: dense %.3f ms, hash %.3f ms"
          % (n, v, cells, 32e-6 * cells, m, dense, hashed))
EOF

python - <<'EOF'
import torch
x = torch.empty(4 << 30, dtype=torch.uint8, device="cuda")
y = torch.empty_like(x)
for _ in range(3):
    y.copy_(x)
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
reps = 20
e0.record()
for _ in range(reps):
    y.copy_(x)
e1.record()
torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / reps
print("device-to-device copy of 4 GiB: %.3f ms = %.0f GB/s (bytes read + written)" % (ms, 2 * x.numel() / (ms * 1e-3) / 1e9))
EOF
