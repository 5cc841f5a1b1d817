// Edge stage of IEGMN_Layer.forward (rigid_docking_model.py:204-237, 263-292), one fused kernel:
//   x_rel = x[src]-x[dst] (fp64) -> 15 RBFs exp(-d^2/1.5^s) -> edge MLP (Linear, LeakyReLU, LayerNorm,
//   Linear) -> coordinate MLP (Linear, LeakyReLU, Linear->1) -> mean over each destination's
//   in-edges of msg (aggr_msg) and of x_rel*phi (x_update) -> x' = eta*x0 + (1-eta)*x + x_update.
// The first Linear of the edge MLP is split: its [h_src | h_dst] columns were applied per NODE
// by the projection stage (Psrc, Pdst(+bias)); only the 27+15 per-edge columns are a GEMM here.
// Per-edge activations never leave the SM.
#include "edge_tile.cuh"

namespace eqd {

struct EdgeSmem : EdgeTileSmem {
  float buf[EQD_TM * EDGE_LD];
  float phi[EQD_TM];
  int rp[EQD_TM + 1];
};

// DROP: training-mode dropout sites 0 (z1) and 1 (z3) of eqd_dropout `dr`, applied before their LeakyReLU.
// CLN: the coordinate LayerNorm coors_mlp.3 of eqd_layer_norms `nm` after coors_mlp.2 (the same statistics code as
// edge_mlp.3), so phi = w4 . LN(LeakyReLU(z3)) + b4.
template <bool DROP, bool CLN>
__global__ void __launch_bounds__(EQD_THREADS, 2)
edge_stage_kernel(eqd_graph g, eqd_layer_params p, const float* __restrict__ proj, const double* __restrict__ x_in,
                  const double* __restrict__ x_orig, float* __restrict__ aggr, double* __restrict__ x_out,
                  int* __restrict__ status, int tn /* destination nodes per tile */, eqd_dropout dr, eqd_layer_norms nm) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  EdgeSmem& s = *reinterpret_cast<EdgeSmem*>(smem_raw);
  const int tid = threadIdx.x, ty = tid >> 3, tx = tid & 7;
  const int pw = 128 + 3 * p.dhp;

  edge_tile_weights<CLN>(s, p, nm, tid);  // once per CTA
  __syncthreads();

  const int ntiles = (g.n_nodes + tn - 1) / tn;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int n0 = tile * tn;
    const int nn = min(tn, g.n_nodes - n0);
    for (int i = tid; i <= nn; i += EQD_THREADS) s.rp[i] = g.row_ptr[n0 + i];
    __syncthreads();
    const int e0 = s.rp[0];
    const int ne = s.rp[nn] - e0;
    if (ne > EQD_TM) {  // in-degree bound violated: flag and skip (uniform branch)
      if (tid == 0) atomicOr(status + g.n_pairs, EQD_STATUS_DEGREE_OVERFLOW);
      __syncthreads();
      continue;
    }

    edge_tile_inputs(s, s.buf, g, x_in, e0, ne, tid);
    __syncthreads();

    // ---- edge_mlp.0: gathered node projections + [he|rbf] GEMM -------------------------------
    float acc[8][8], accx[8];
    edge_tile_z1<DROP>(acc, accx, s, s.buf, proj, pw, dr, e0, ty, tx);
    lrelu_layernorm<false>(acc, accx, s.ln_g, s.ln_b, 64, p.leaky_slope, tx);  // edge_mlp.2-3
    __syncthreads();  // everyone is done reading the [he|rbf] operand
    store_tile_smem<false>(s.buf, EDGE_LD, acc, accx, ty, tx);
    __syncthreads();

    // ---- edge_mlp.4 -> msg --------------------------------------------------------------------
    acc_set_bias(acc, s.b2, tx);
    gemm_nn<false>(acc, accx, s.buf + ty * 8 * EDGE_LD, EDGE_LD, s.w2, 64, 64, tx);
    __syncthreads();
    store_tile_smem<false>(s.buf, EDGE_LD, acc, accx, ty, tx);  // msg tile (A of coors_mlp, source of aggr)
    __syncthreads();

    // ---- coors_mlp: Linear, LeakyReLU, (LayerNorm,) Linear(64->1) -> phi ------------------------
    acc_set_bias(acc, s.b3, tx);
    gemm_nn<false>(acc, accx, s.buf + ty * 8 * EDGE_LD, EDGE_LD, s.w3, 64, 64, tx);
    if (DROP) dropout_tile<false>(acc, accx, dr, 1, e0 + ty * 8, tx);
    if (CLN) lrelu_layernorm<false>(acc, accx, s.cln_g, s.cln_b, 64, p.leaky_slope, tx);  // coors_mlp.2-3
    {
      float w4r[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) w4r[j] = s.w4[col_nn(tx, j)];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float v = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) v = fmaf(CLN ? acc[i][j] : lrelu(acc[i][j], p.leaky_slope), w4r[j], v);
        v = row_sum8(v);
        if (tx == 0) s.phi[ty * 8 + i] = v + p.b_coor2;
      }
    }
    __syncthreads();

    // ---- mean aggregation at the destination (:274-283) + coordinate update (:286-292) ----------
    for (int o = tid; o < nn * 64; o += EQD_THREADS) {
      int nd = o >> 6, c = o & 63;
      int rs = s.rp[nd] - e0, re = s.rp[nd + 1] - e0;
      float sum = 0.f;
      for (int r = rs; r < re; ++r) sum += s.buf[r * EDGE_LD + c];
      int deg = re - rs;
      aggr[(long)(n0 + nd) * 64 + c] = deg > 0 ? sum / (float)deg : 0.f;
    }
    for (int o = tid; o < nn * 3; o += EQD_THREADS) {
      int nd = o / 3, comp = o - nd * 3;
      int rs = s.rp[nd] - e0, re = s.rp[nd + 1] - e0;
      double sum = 0.0;
      for (int r = rs; r < re; ++r) sum += s.xrel[r * 3 + comp] * (double)s.phi[r];  // x_rel * phi :264
      int deg = re - rs;
      double upd = deg > 0 ? sum / (double)deg : 0.0;
      long gi = (long)(n0 + nd) * 3 + comp;
      double eta = (double)p.x_connection_init;
      x_out[gi] = eta * x_orig[gi] + (1.0 - eta) * x_in[gi] + upd;
    }
    __syncthreads();
  }
}

template <bool DROP, bool CLN>
static int launch_edge_stage(const eqd_graph* g, const eqd_layer* p_l, const float* proj, const double* x_in,
                             const double* x_orig, float* aggr, double* x_out, int32_t* status, int tn, int grid,
                             void* stream) {
  const size_t smem = sizeof(EdgeSmem);
  EQD_SET_SMEM((edge_stage_kernel<DROP, CLN>), smem);
  edge_stage_kernel<DROP, CLN><<<grid, EQD_THREADS, smem, (cudaStream_t)stream>>>(*g, p_l->dev, proj, x_in, x_orig, aggr,
                                                                                  x_out, status, tn, p_l->dropout, p_l->norms);
  EQD_CUDA_LAUNCH_CHECK();
  return EQD_OK;
}

}  // namespace eqd

extern "C" int eqd_edge_stage_ffma(const eqd_graph* g, const eqd_layer* p_l, const float* proj, const double* x_in,
                              const double* x_orig, float* aggr, double* x_out, int32_t* status, void* stream) {
  const eqd_layer_params* p = p_l ? &p_l->dev : nullptr;
  if (!g || !p || !proj || !x_in || !x_orig || !aggr || !x_out || !status) return EQD_ERR_BAD_ARG;
  const int cln = eqd_coors_ln(p_l);
  if (cln < 0) return EQD_ERR_BAD_ARG;
  if (g->max_in_degree < 1 || g->max_in_degree > EQD_TM) return EQD_ERR_UNSUPPORTED;
  if (!(p->leaky_slope >= 0.f && p->leaky_slope <= 1.f)) return EQD_ERR_UNSUPPORTED;  // lrelu() = max(v, slope*v)
  if (g->n_nodes <= 0) return EQD_OK;
  int tn = EQD_TM / g->max_in_degree;
  if (tn > EQD_TM) tn = EQD_TM;
  int ntiles = (g->n_nodes + tn - 1) / tn;
  int grid = ntiles < EQD_SMS * 2 ? ntiles : EQD_SMS * 2;
  const bool drop = p_l->dropout.p > 0.f;
  if (cln)
    return drop ? eqd::launch_edge_stage<true, true>(g, p_l, proj, x_in, x_orig, aggr, x_out, status, tn, grid, stream)
                : eqd::launch_edge_stage<false, true>(g, p_l, proj, x_in, x_orig, aggr, x_out, status, tn, grid, stream);
  return drop ? eqd::launch_edge_stage<true, false>(g, p_l, proj, x_in, x_orig, aggr, x_out, status, tn, grid, stream)
              : eqd::launch_edge_stage<false, false>(g, p_l, proj, x_in, x_orig, aggr, x_out, status, tn, grid, stream);
}
