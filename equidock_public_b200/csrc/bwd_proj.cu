// Backward of the per-node projections (the node-side split of edge_mlp.0 plus att_mlp_Q/K/V,
// rigid_docking_model.py:130-140, 186, 229-231, 247-256) and of the input embedding (:459-471).
//   bwd_proj_kernel : dh[n] += dP[n][0 : pw] . Wproj^T     (dP = [dPsrc | dPdst | dQpre | dKpre | dV])
//   bwd_embed_kernel: d residue_emb_layer.weight[r] = sum over nodes with residue r of (dh0_acc[n] + dh_layer0[n])[0:64]
// Restated in oracle/backward_manual.py::proj_bwd / full_backward.
#include "bwd_common.cuh"

namespace eqd {

template <bool EXTRA>
__global__ void __launch_bounds__(EQD_THREADS)
bwd_proj_kernel(int n_nodes, const float* __restrict__ w_projT /*[pw][dhp]*/, const float* __restrict__ dP,
                float* __restrict__ dh /*[n][dhp], accumulated into*/) {
  constexpr int DHP = EXTRA ? 72 : 64;
  constexpr int LD = 68;
  extern __shared__ __align__(16) float smem[];
  float* bufA = smem;                  // [128][68]: one 64-column chunk of dP
  float* wbuf = smem + EQD_TM * LD;
  const int tid = threadIdx.x, ty = tid >> 3, tx = tid & 7;
  const int pw = 128 + 3 * DHP;
  const int ntiles = (n_nodes + EQD_TM - 1) / EQD_TM;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int node0 = tile * EQD_TM;
    const int nvalid = min(EQD_TM, n_nodes - node0);
    float acc[8][8], accx[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      accx[i] = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
    }
    for (int k0 = 0; k0 < pw; k0 += 64) {
      const int kc = min(64, pw - k0);
      tile_load_async(bufA, LD, dP + (long)node0 * pw + k0, pw, EQD_TM, nvalid, kc, tid);
      cp_async_commit();
      cp_async_wait<0>();
      __syncthreads();
      gemm_nn_stream<EXTRA>(acc, accx, bufA + ty * 8 * LD, LD, kc, w_projT + (long)k0 * DHP, DHP, DHP, wbuf, tid);
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int r = ty * 8 + i;
      if (r < nvalid) {
        float* o = dh + (long)(node0 + r) * DHP + tx * 4;
        float4 a = *reinterpret_cast<float4*>(o), b = *reinterpret_cast<float4*>(o + 32);
        *reinterpret_cast<float4*>(o) = make_float4(a.x + acc[i][0], a.y + acc[i][1], a.z + acc[i][2], a.w + acc[i][3]);
        *reinterpret_cast<float4*>(o + 32) = make_float4(b.x + acc[i][4], b.y + acc[i][5], b.z + acc[i][6], b.w + acc[i][7]);
        if (EXTRA) dh[(long)(node0 + r) * DHP + 64 + tx] += accx[i];
      }
    }
    __syncthreads();
  }
}

// grid = 21 residue types; thread (c = tid & 63, part = tid >> 6): fixed-order strided sums, then a fixed-order merge.
__global__ void bwd_embed_kernel(eqd_graph g, const float* __restrict__ res_l, const float* __restrict__ res_r,
                                 const float* __restrict__ dh0_acc /*[n][72]*/, const float* __restrict__ dh_l0 /*[n][72]*/,
                                 float* __restrict__ demb /*[21][64]*/) {
  __shared__ float sh[4][64];
  const int r = blockIdx.x, c = threadIdx.x & 63, part = threadIdx.x >> 6;
  float t = 0.f;
  for (int n = part; n < g.n_nodes; n += 4) {
    const bool lig = n < g.n_lig_nodes;
    int rr = (int)(lig ? res_l[n] : res_r[n - g.n_lig_nodes]);
    rr = min(max(rr, 0), EQD_N_RES_TYPES - 1);
    if (rr == r) t += dh0_acc[(long)n * EQD_H0_PAD + c] + dh_l0[(long)n * EQD_H0_PAD + c];
  }
  sh[part][c] = t;
  __syncthreads();
  if (part == 0) demb[r * 64 + c] += (sh[0][c] + sh[1][c]) + (sh[2][c] + sh[3][c]);
}

}  // namespace eqd

extern "C" int eqd_bwd_project(const eqd_graph* g, const eqd_layer* p_l, const float* w_projT, const float* dP,
                               float* dh, void* stream) {
  const eqd_layer_params* p = p_l ? &p_l->dev : nullptr;
  if (!g || !p || !w_projT || !dP || !dh) return EQD_ERR_BAD_ARG;
  const bool extra = (p->dh == 69 && p->dhp == 72);
  if (!extra && !(p->dh == 64 && p->dhp == 64)) return EQD_ERR_UNSUPPORTED;
  if (g->n_nodes <= 0) return EQD_OK;
  const int ntiles = (g->n_nodes + EQD_TM - 1) / EQD_TM;
  const int grid = ntiles < EQD_SMS * 2 ? ntiles : EQD_SMS * 2;
  const size_t smem = (size_t)(EQD_TM * 68 + 2 * EQD_WCHUNK * EQD_WLD) * sizeof(float);
  if (extra) {
    EQD_SET_SMEM((eqd::bwd_proj_kernel<true>), smem);
    eqd::bwd_proj_kernel<true><<<grid, EQD_THREADS, smem, (cudaStream_t)stream>>>(g->n_nodes, w_projT, dP, dh);
  } else {
    EQD_SET_SMEM((eqd::bwd_proj_kernel<false>), smem);
    eqd::bwd_proj_kernel<false><<<grid, EQD_THREADS, smem, (cudaStream_t)stream>>>(g->n_nodes, w_projT, dP, dh);
  }
  EQD_CUDA_LAUNCH_CHECK();
  return EQD_OK;
}

extern "C" int eqd_bwd_embed(const eqd_graph* g, const float* res_lig, const float* res_rec, const float* dh0_acc,
                             const float* dh_layer0, float* demb, void* stream) {
  if (!g || !res_lig || !res_rec || !dh0_acc || !dh_layer0 || !demb) return EQD_ERR_BAD_ARG;
  if (g->n_nodes <= 0) return EQD_OK;
  eqd::bwd_embed_kernel<<<EQD_N_RES_TYPES, 256, 0, (cudaStream_t)stream>>>(*g, res_lig, res_rec, dh0_acc, dh_layer0, demb);
  EQD_CUDA_LAUNCH_CHECK();
  return EQD_OK;
}
