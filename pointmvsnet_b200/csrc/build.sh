#!/usr/bin/env bash
# Builds libpmvs_b200.so (sm_90a only) next to the Python package.
set -euo pipefail
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
OUT="${PMVS_OUT:-${HERE}/../libpmvs_b200.so}"   # PMVS_OUT=<path> builds a side copy (experimental flags)
NVCC="${NVCC:-/usr/local/cuda/bin/nvcc}"
FLAGS=(-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -shared
       --expt-relaxed-constexpr -Xptxas -v)
"${NVCC}" "${FLAGS[@]}" -o "${OUT}" "${HERE}"/api.cu "${HERE}"/knn3d.cu "${HERE}"/fetch.cu "${HERE}"/edgeconv.cu "${HERE}"/gemm_tc.cu "${HERE}"/edge_tile.cu "${HERE}"/gemm_ws.cu "${HERE}"/gather_det.cu "${HERE}"/edge_bwd.cu "${HERE}"/flow_bwd.cu "${HERE}"/cost_volume_bwd.cu "${HERE}"/fetch_bwd_det.cu "${HERE}"/depth_fusion.cu "${HERE}"/consistency_fusion.cu "${HERE}"/tsdf.cu "${HERE}"/mesh.cu "${HERE}"/cloud_eval.cu "${HERE}"/volume_conv.cu "${HERE}"/volume_conv_bwd.cu "${HERE}"/image_conv.cu "${HERE}"/image_conv_bwd.cu "${HERE}"/depth_loss.cu "${HERE}"/flow_eval.cu "${HERE}"/prepare_views.cu "${HERE}"/prob_filter.cu "$@"
echo "built ${OUT}"
