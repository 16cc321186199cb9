#!/bin/bash
# Run on the GPU box (under gpurun): launch list + one full ncu capture of the bucket-accumulate kernel.
# Usage: tools/profile.sh <round-tag>
set -u
TAG=${1:-r02z}
mkdir -p gpurun_out
export B2K_SKIP_CPU_BASELINE=1
export B2K_SKIP_PAIRINGS=1
export B2K_SKIP_SECTIONS=1
export B2K_SKIP_SUSTAINED=1
# every launch with its device time (cold-cache, serialised: compare SHARES, not absolutes)
ncu --metrics gpu__time_duration.sum --clock-control none -c 400 --csv --log-file gpurun_out/launches_${TAG}.csv \
    python bench.py --steps 2 --warmup 3 > gpurun_out/bench_under_ncu_${TAG}.log 2>&1
python tools/summarize_launches.py gpurun_out/launches_${TAG}.csv > gpurun_out/${TAG}_launches_summary.txt 2>&1
# the bucket-accumulate pass of ONE MSM, once: the three kernels of every affine pair-tree round + the XYZZ slices
# (NK = 3 R + 1 launches per MSM; skip the first 3 MSMs)
NK=${B2K_PROFILE_PASS_KERNELS:-10}
ncu --set full --clock-control none --import-source on -k "regex:k_pt_forward|k_pt_backward|k_msm_accumulate_slices" -s $((3 * NK)) -c $NK \
    -o gpurun_out/accumulate_${TAG} -f python bench.py --steps 1 --warmup 3 --contexts 1 > gpurun_out/ncu_full_${TAG}.log 2>&1
# gpurun_out/ travels back only below 64 MiB: keep the text pages, drop the report
ncu -i gpurun_out/accumulate_${TAG}.ncu-rep --page details > gpurun_out/${TAG}_accumulate_ncu_details.txt 2>&1
ncu -i gpurun_out/accumulate_${TAG}.ncu-rep --page raw --csv > gpurun_out/${TAG}_accumulate_ncu_raw.csv 2>&1
python tools/ncu_traffic.py gpurun_out/${TAG}_accumulate_ncu_raw.csv ${TAG} > gpurun_out/accumulate_traffic.json 2> gpurun_out/ncu_traffic_${TAG}.err
rm -f gpurun_out/accumulate_${TAG}.ncu-rep
# pairing kernel: one full capture AT THE BENCHMARK SIZE (65 536 checks, the batch bench.py times)
cat > /tmp/pair_probe.py <<'PY'
import sys
sys.path.insert(0, '.')
import torch
from kyber_b200 import Engine
from oracle import bls12381 as o
eng = Engine(0); n = 65536
a1 = torch.frombuffer(bytearray(o.g1_to_affine_bytes(o.g1_mul(12345)) * n), dtype=torch.uint8).cuda()
a2 = torch.frombuffer(bytearray(o.g2_to_affine_bytes(o.g2_mul(6789)) * n), dtype=torch.uint8).cuda()
ok = torch.empty(n, dtype=torch.uint8, device='cuda')
eng._check(eng.lib.b2k_bls12381_pairing_check_dev(eng.h, n, a1.data_ptr(), a2.data_ptr(), a1.data_ptr(), a2.data_ptr(), ok.data_ptr()))
eng.synchronize(); print(int(ok.sum()))
PY
ncu --set full --clock-control none --import-source on -k regex:k_bls_pairing_check -c 1 \
    -o gpurun_out/pairing_check_${TAG} -f python /tmp/pair_probe.py > gpurun_out/ncu_pairing_${TAG}.log 2>&1
ncu -i gpurun_out/pairing_check_${TAG}.ncu-rep --page details > gpurun_out/${TAG}_pairing_check_ncu_details.txt 2>&1
ncu -i gpurun_out/pairing_check_${TAG}.ncu-rep --page raw --csv > gpurun_out/${TAG}_pairing_check_ncu_raw.csv 2>&1
rm -f gpurun_out/pairing_check_${TAG}.ncu-rep
ls -la gpurun_out
