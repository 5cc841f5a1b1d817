// Input stage (IEGMN.forward, rigid_docking_model.py:452-471) and the per-layer node projections.
#include "common.cuh"

namespace eqd {

// One thread per (node, 4-channel group): h0[n] = [emb[res] | log(mu) | 0], x64[n] = coords.
__global__ void embed_kernel(eqd_graph g, const float* __restrict__ emb, const float* __restrict__ res_l,
                             const float* __restrict__ res_r, const float* __restrict__ mu_l,
                             const float* __restrict__ mu_r, const float* __restrict__ x_l,
                             const float* __restrict__ x_r, float* __restrict__ h0, double* __restrict__ x64,
                             int32_t* __restrict__ status) {
  const int per_node = EQD_H0_PAD / 4;  // 18 float4 per node
  long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  long total = (long)g.n_nodes * per_node;
  if (idx >= total) return;
  int n = (int)(idx / per_node), q = (int)(idx - (long)n * per_node);
  bool lig = n < g.n_lig_nodes;
  int ln = lig ? n : n - g.n_lig_nodes;
  float4 v;
  if (q < 16) {
    // .view(-1).long() truncation of the fp32-encoded residue index (:460)
    const float rf = lig ? res_l[ln] : res_r[ln];
    int r = (int)rf;
    // nn.Embedding raises on an index outside [0, 21): flag it (the host raises in resolve_status); the clamp only
    // keeps this launch memory-safe.  NaN converts to 0 here but to INT64_MIN under .long(): it is out of range too.
    if ((rf != rf || r < 0 || r >= EQD_N_RES_TYPES) && status && q == 0) atomicOr(status + g.n_pairs, EQD_STATUS_BAD_RESIDUE);
    r = min(max(r, 0), EQD_N_RES_TYPES - 1);
    v = *reinterpret_cast<const float4*>(emb + r * 64 + q * 4);
  } else {
    const float* mu = (lig ? mu_l : mu_r) + (long)ln * 5;
    if (q == 16) {
      v = make_float4(logf(mu[0]), logf(mu[1]), logf(mu[2]), logf(mu[3]));  // torch.log(mu_r_norm) :469
    } else {
      v = make_float4(logf(mu[4]), 0.f, 0.f, 0.f);
      const float* xs = (lig ? x_l : x_r) + (long)ln * 3;  // ligand 'new_x', receptor 'x' (:455-456)
      x64[(long)n * 3 + 0] = (double)xs[0];
      x64[(long)n * 3 + 1] = (double)xs[1];
      x64[(long)n * 3 + 2] = (double)xs[2];
    }
  }
  *reinterpret_cast<float4*>(h0 + (long)n * EQD_H0_PAD + q * 4) = v;
}

// Stand-alone projection of h (layer 0: h = h0, K = 72).  Later layers get theirs fused into the
// previous layer's node stage.
template <bool EXTRA>
__global__ void __launch_bounds__(EQD_THREADS) project_kernel(eqd_graph g, eqd_layer_params p,
                                                              const float* __restrict__ h, int ldh,
                                                              float* __restrict__ proj) {
  extern __shared__ __align__(16) float smem[];
  const int lda = p.dhp + 4;
  float* A = smem;                    // [128][lda]
  float* wbuf = smem + EQD_TM * lda;  // 2*32*72
  const int tid = threadIdx.x;
  const int ntiles = (g.n_nodes + EQD_TM - 1) / EQD_TM;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    int node0 = tile * EQD_TM;
    int nvalid = min(EQD_TM, g.n_nodes - node0);
    tile_load_async(A, lda, h + (long)node0 * ldh, ldh, EQD_TM, nvalid, p.dhp, tid);
    cp_async_commit();
    cp_async_wait<0>();
    __syncthreads();
    project_tile<EXTRA>(A, lda, p, proj, node0, nvalid, wbuf, tid);
    __syncthreads();
  }
}

}  // namespace eqd

extern "C" int eqd_embed_checked(const eqd_graph* g, const float* emb, const float* res_feat_lig,
                                 const float* res_feat_rec, const float* mu_lig, const float* mu_rec, const float* x_lig,
                                 const float* x_rec, float* h0, double* x64, int32_t* status, void* stream) {
  if (!g || !emb || !h0 || !x64) return EQD_ERR_BAD_ARG;
  if (g->n_nodes <= 0) return EQD_OK;
  long total = (long)g->n_nodes * (EQD_H0_PAD / 4);
  int block = 256;
  long grid = (total + block - 1) / block;
  eqd::embed_kernel<<<(unsigned)grid, block, 0, (cudaStream_t)stream>>>(*g, emb, res_feat_lig, res_feat_rec, mu_lig,
                                                                        mu_rec, x_lig, x_rec, h0, x64, status);
  EQD_CUDA_LAUNCH_CHECK();
  return EQD_OK;
}

extern "C" int eqd_embed(const eqd_graph* g, const float* emb, const float* res_feat_lig, const float* res_feat_rec,
                         const float* mu_lig, const float* mu_rec, const float* x_lig, const float* x_rec, float* h0,
                         double* x64, void* stream) {
  return eqd_embed_checked(g, emb, res_feat_lig, res_feat_rec, mu_lig, mu_rec, x_lig, x_rec, h0, x64, nullptr, stream);
}

extern "C" int eqd_project(const eqd_graph* g, const eqd_layer* p_l, const float* h, int32_t ldh, float* proj,
                           void* stream) {
  const eqd_layer_params* p = p_l ? &p_l->dev : nullptr;
  if (!g || !p || !h || !proj) return EQD_ERR_BAD_ARG;
  if (!((p->dh == 64 && p->dhp == 64) || (p->dh == 69 && p->dhp == 72))) return EQD_ERR_UNSUPPORTED;
  if (!(p->leaky_slope >= 0.f && p->leaky_slope <= 1.f)) return EQD_ERR_UNSUPPORTED;  // lrelu() = max(v, slope*v)
  if (g->n_nodes <= 0) return EQD_OK;
  int ntiles = (g->n_nodes + EQD_TM - 1) / EQD_TM;
  size_t smem = (size_t)(EQD_TM * (p->dhp + 4) + 2 * EQD_WCHUNK * EQD_WLD) * sizeof(float);
  int grid = ntiles < EQD_SMS * 4 ? ntiles : EQD_SMS * 4;
  if (p->dhp == 72) {
    EQD_SET_SMEM((eqd::project_kernel<true>), smem);
    eqd::project_kernel<true><<<grid, EQD_THREADS, smem, (cudaStream_t)stream>>>(*g, *p, h, ldh, proj);
  } else {
    EQD_SET_SMEM((eqd::project_kernel<false>), smem);
    eqd::project_kernel<false><<<grid, EQD_THREADS, smem, (cudaStream_t)stream>>>(*g, *p, h, ldh, proj);
  }
  EQD_CUDA_LAUNCH_CHECK();
  return EQD_OK;
}
