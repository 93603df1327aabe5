#!/bin/bash
# Captures the exact stdout / stderr / exit code of the READ-ONLY nvidia-smi invocations the reference's detach side
# parses, on a real box, so csrc/nvml_ops.cpp can be pinned to them.  Nothing here changes the GPU's state.
OUT=${1:?usage: smi_texts.sh OUTPUT_DIR}; mkdir -p "$OUT"
BUS=$(nvidia-smi --query-gpu=pci.bus_id --format=csv,noheader,nounits | head -1)
SHORT=${BUS#0000}
run() { local tag=$1; shift; "$@" > $OUT/$tag.out 2> $OUT/$tag.err; echo $? > $OUT/$tag.rc; }
run drain_q_long   nvidia-smi drain -p "$BUS" -q
run drain_q_short  nvidia-smi drain -p "$SHORT" -q
run drain_q_lower  nvidia-smi drain -p "$(echo $SHORT | tr A-F a-f)" -q
run drain_q_bad    nvidia-smi drain -p 0000:FE:00.0 -q
run drain_q_junk   nvidia-smi drain -p junk -q
run apps_idle      nvidia-smi --query-compute-apps=gpu_uuid,process_name --format=csv,noheader,nounits
python - <<'PY' &
import torch, time
x = torch.zeros(1 << 20, device="cuda"); torch.cuda.synchronize(); time.sleep(8)
PY
sleep 5
run apps_busy      nvidia-smi --query-compute-apps=gpu_uuid,process_name,pid --format=csv,noheader,nounits
run apps_busy2     nvidia-smi --query-compute-apps=gpu_uuid,process_name --format=csv,noheader,nounits
ps -eo pid,comm,args | grep -i python | head -5 > $OUT/ps.txt
wait
echo "$BUS" > $OUT/bus.txt
for f in $OUT/*; do echo "== $f"; cat -A $f | head -5; done
