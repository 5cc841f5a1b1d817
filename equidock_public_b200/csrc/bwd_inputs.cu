// Gradients with respect to the graph's input tensors (ligand new_x, receptor x, both mu_r_norm, both edge types' he):
// what the reference's autograd hands to any module upstream of rigid_docking_model.py.  Only launched when a caller asks
// for them; the parameter-gradient path never reads their outputs.
//   bwd_layer_inputs_kernel: once per layer, after eqd_bwd_edge.  dhe += dz1 . w_edge1[0:27]^T (he enters every layer
//                            through edge_mlp.0, :229-231) and dx_orig += eta dx_out (x_orig = the input coordinates in
//                            every layer, :286-292; eqd_bwd_edge_gather keeps only the (1 - eta) share).
//   bwd_inputs_kernel      : once after the layer loop.  d mu_r_norm = dh0[64:69] / mu_r_norm (h0 = [emb | log mu],
//                            :468-471); d x_in = dx_layer0 + dx_orig (+ T^T dcoors for a ligand node: ligand_out =
//                            T new_x + b, :657-665).
// No atomics: every output element is owned by one thread and accumulated in layer order.
#include "bwd_common.cuh"

namespace eqd {

#define LI_LD 68   // dz1 tile row stride (floats): conflict-free float4 row reads

// grid-stride over 128-edge tiles; thread t owns edge row t of a tile.  The dz1 tile buffer is reused to stage the
// [128][27] result so that the read-modify-write of dhe (contiguous for a tile) is coalesced.
__global__ void __launch_bounds__(EQD_THREADS)
bwd_layer_inputs_kernel(int n_edges, int n_nodes, const float* __restrict__ w_edge1 /*[44][64]*/,
                        const float* __restrict__ dz1 /*[E][64]*/, const double* __restrict__ dx_out, double eta,
                        float* __restrict__ dhe /*[E][27]*/, double* __restrict__ dx_orig) {
  __shared__ __align__(16) float ws[EQD_EDGE_FEATS * 64];
  __shared__ __align__(16) float zs[EQD_TM * LI_LD];
  const int tid = threadIdx.x;
  for (int i = tid; i < EQD_EDGE_FEATS * 64; i += EQD_THREADS) ws[i] = w_edge1[i];
  const int ntiles = (n_edges + EQD_TM - 1) / EQD_TM;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const long e0 = (long)tile * EQD_TM;
    const int nvalid = (int)min((long)EQD_TM, n_edges - e0);
    tile_load_async(zs, LI_LD, dz1 + e0 * 64, 64, EQD_TM, nvalid, 64, tid);
    cp_async_commit();
    cp_async_wait<0>();
    __syncthreads();
    float acc[EQD_EDGE_FEATS];
#pragma unroll
    for (int f = 0; f < EQD_EDGE_FEATS; ++f) acc[f] = 0.f;
    const float* z = zs + tid * LI_LD;
#pragma unroll 2
    for (int k = 0; k < 64; k += 4) {
      const float4 a = *reinterpret_cast<const float4*>(z + k);
#pragma unroll
      for (int f = 0; f < EQD_EDGE_FEATS; ++f) {
        const float4 w = *reinterpret_cast<const float4*>(ws + f * 64 + k);
        acc[f] = fmaf(a.x, w.x, acc[f]);
        acc[f] = fmaf(a.y, w.y, acc[f]);
        acc[f] = fmaf(a.z, w.z, acc[f]);
        acc[f] = fmaf(a.w, w.w, acc[f]);
      }
    }
    __syncthreads();                       // every row of zs has been read: reuse it as the [128][27] staging tile
#pragma unroll
    for (int f = 0; f < EQD_EDGE_FEATS; ++f) zs[tid * EQD_EDGE_FEATS + f] = acc[f];
    __syncthreads();
    float* out = dhe + e0 * EQD_EDGE_FEATS;
    for (int i = tid; i < nvalid * EQD_EDGE_FEATS; i += EQD_THREADS) out[i] += zs[i];
    __syncthreads();
  }
  for (long i = (long)blockIdx.x * EQD_THREADS + tid; i < 3L * n_nodes; i += (long)gridDim.x * EQD_THREADS)
    dx_orig[i] += eta * dx_out[i];
}

// one thread per node
__global__ void bwd_inputs_kernel(eqd_graph g, const float* __restrict__ dh0_acc, const float* __restrict__ dh_l0,
                                  const float* __restrict__ mu_lig, const float* __restrict__ mu_rec,
                                  const double* __restrict__ dx_l0, const double* __restrict__ dx_orig,
                                  const float* __restrict__ rot, const float* __restrict__ dcoors,
                                  float* __restrict__ dmu, double* __restrict__ dx) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= g.n_nodes) return;
  const bool lig = n < g.n_lig_nodes;
  const float* mu = lig ? mu_lig + (long)n * 5 : mu_rec + (long)(n - g.n_lig_nodes) * 5;
#pragma unroll
  for (int c = 0; c < 5; ++c)
    dmu[(long)n * 5 + c] = (dh0_acc[(long)n * EQD_H0_PAD + 64 + c] + dh_l0[(long)n * EQD_H0_PAD + 64 + c]) / mu[c];
  double gx[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) gx[r] = dx_l0[(long)n * 3 + r] + dx_orig[(long)n * 3 + r];
  if (lig && dcoors) {
    int lo = 0, hi = g.n_pairs - 1;        // the pair b with seg_ptr[b] <= n < seg_ptr[b + 1]
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (g.seg_ptr[mid] <= n) lo = mid; else hi = mid - 1;
    }
    const float* T = rot + (long)lo * 9;
    const double d0 = dcoors[(long)n * 3], d1 = dcoors[(long)n * 3 + 1], d2 = dcoors[(long)n * 3 + 2];
#pragma unroll
    for (int c = 0; c < 3; ++c) gx[c] += (double)T[c] * d0 + (double)T[3 + c] * d1 + (double)T[6 + c] * d2;
  }
#pragma unroll
  for (int r = 0; r < 3; ++r) dx[(long)n * 3 + r] = gx[r];
}

}  // namespace eqd

extern "C" int eqd_bwd_layer_inputs(const eqd_graph* g, const eqd_layer* p_l, const float* dz1, const double* dx_out,
                                    float* dhe, double* dx_orig, void* stream) {
  const eqd_layer_params* p = p_l ? &p_l->dev : nullptr;
  if (!g || !p || !p->w_edge1 || !dz1 || !dx_out || !dhe || !dx_orig) return EQD_ERR_BAD_ARG;
  if (g->n_edges < 0 || g->n_nodes < 0) return EQD_ERR_BAD_ARG;
  if (reinterpret_cast<uintptr_t>(dz1) & 15) return EQD_ERR_BAD_ARG;
  const long ntiles = (g->n_edges + EQD_TM - 1) / EQD_TM;
  const long nblocks = (3L * g->n_nodes + EQD_THREADS - 1) / EQD_THREADS;
  long grid = ntiles > nblocks ? ntiles : nblocks;
  if (grid > EQD_SMS * 4) grid = EQD_SMS * 4;
  if (grid == 0) return EQD_OK;
  eqd::bwd_layer_inputs_kernel<<<(unsigned)grid, EQD_THREADS, 0, (cudaStream_t)stream>>>(
      g->n_edges, g->n_nodes, p->w_edge1, dz1, dx_out, (double)p->x_connection_init, dhe, dx_orig);
  EQD_CUDA_LAUNCH_CHECK();
  return EQD_OK;
}

extern "C" int eqd_bwd_inputs(const eqd_graph* g, const float* dh0_acc, const float* dh_layer0, const float* mu_lig,
                              const float* mu_rec, const double* dx_layer0, const double* dx_orig, const float* rot,
                              const float* dcoors, float* dmu, double* dx, void* stream) {
  if (!g || !dh0_acc || !dh_layer0 || !mu_lig || !mu_rec || !dx_layer0 || !dx_orig || !rot || !dmu || !dx)
    return EQD_ERR_BAD_ARG;
  if (g->n_nodes <= 0) return EQD_OK;
  eqd::bwd_inputs_kernel<<<(unsigned)((g->n_nodes + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      *g, dh0_acc, dh_layer0, mu_lig, mu_rec, dx_layer0, dx_orig, rot, dcoors, dmu, dx);
  EQD_CUDA_LAUNCH_CHECK();
  return EQD_OK;
}
