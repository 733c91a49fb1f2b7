#!/usr/bin/env bash
# Builds libsmaat_b200.so in-tree for sm_90a (H100).  nvcc cross-compiles without a GPU.
set -euo pipefail
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
OUT=../libsmaat_b200.so
FLAGS=(-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC,-O2,-Wall
       -Xptxas -v -cudart static)
SRCS=(runtime.cu dw3x3.cu dw3x3_small.cu pw1x1.cu pw1x1_simt.cu pw1x1_tc.cu pw1x1_wgrad_tc.cu dsconv_fused.cu glue.cu upsample.cu cbam.cu bn.cu backward.cu bn_bwd.cu loss_metrics.cu ce_metrics.cu dw3x3_bwd.cu cbam_bwd.cu optim.cu convt.cu conv3x3_tc.cu conv3x3_wgrad_tc.cu conv3x3_simt.cu voc_augment.cu datasets.cu)
mkdir -p ../../build
# objects built with other flags (another architecture, say) are rebuilt
if [[ "$(cat ../../build/.flags 2>/dev/null || true)" != "${FLAGS[*]}" ]]; then rm -f ../../build/*.o; echo "${FLAGS[*]}" > ../../build/.flags; fi
OBJS=()
pids=()
for s in "${SRCS[@]}"; do
  o=../../build/${s%.cu}.o
  OBJS+=("$o")
  if [[ ! -f "$o" || "$s" -nt "$o" || common.cuh -nt "$o" || tc_common.cuh -nt "$o" || wgmma.cuh -nt "$o" || ../../include/smaat_b200.h -nt "$o" ]]; then
    ( "$NVCC" "${FLAGS[@]}" -c "$s" -o "$o" > "../../build/${s%.cu}.log" 2>&1 || { cat "../../build/${s%.cu}.log"; exit 1; } ) &
    pids+=($!)
  fi
done
for p in "${pids[@]:-}"; do [[ -n "$p" ]] && wait "$p"; done
"$NVCC" -shared -cudart static -o "$OUT" "${OBJS[@]}"
echo "built $(realpath $OUT)"
