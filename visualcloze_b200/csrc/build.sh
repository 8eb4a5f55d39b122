#!/usr/bin/env bash
# Builds visualcloze_b200/libvcb200.so in-tree for sm_90a (cross-compiles without a GPU).
set -euo pipefail
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
OUT="${HERE}/../libvcb200.so"
NVCC="${NVCC:-/usr/local/cuda/bin/nvcc}"
FLAGS=(-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 --expt-relaxed-constexpr
       -Xcompiler -fPIC -Xcompiler -Wall -shared)
if [[ "${VCB_PTXAS_V:-0}" == "1" ]]; then FLAGS+=(-Xptxas -v); fi
SRCS=("${HERE}/capi.cu")
[[ -f "${HERE}/flux_engine.cu" ]] && SRCS+=("${HERE}/flux_engine.cu")
[[ -f "${HERE}/vae.cu" ]] && SRCS+=("${HERE}/vae.cu")
[[ -f "${HERE}/text_encoders.cu" ]] && SRCS+=("${HERE}/text_encoders.cu")
"${NVCC}" "${FLAGS[@]}" -o "${OUT}" "${SRCS[@]}"
echo "built ${OUT}"
