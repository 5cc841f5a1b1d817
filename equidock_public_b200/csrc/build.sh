#!/usr/bin/env bash
# Builds the C-ABI shared library in-tree (equidock_public_b200/libeqd_iegmn.so) for sm_90a (H100).
set -euo pipefail
here="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
out="${here}/../libeqd_iegmn.so"
nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 \
     -Xcompiler -fPIC -shared ${EQD_NVCC_EXTRA:-} \
     -o "${out}" "${here}"/embed_project.cu "${here}"/edge_stage.cu "${here}"/edge_stage_tc.cu "${here}"/proj_tc.cu "${here}"/node_mlp_tc.cu "${here}"/attn_tc.cu "${here}"/node_stage.cu "${here}"/head.cu "${here}"/forward.cu "${here}"/bwd_reduce.cu "${here}"/bwd_node.cu "${here}"/bwd_edge.cu "${here}"/bwd_attn.cu "${here}"/bwd_proj.cu "${here}"/bwd_inputs.cu "${here}"/losses.cu "${here}"/graph_build.cu "${here}"/batch_assemble.cu
echo "built ${out}"
