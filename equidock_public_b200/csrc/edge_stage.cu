// Edge stage of IEGMN_Layer.forward (rigid_docking_model.py:204-237, 263-292), one fused kernel:
//   x_rel = x[src]-x[dst] (fp64) -> 15 RBFs exp(-d^2/1.5^s) -> edge MLP (Linear, LeakyReLU, LayerNorm,
//   Linear) -> coordinate MLP (Linear, LeakyReLU, Linear->1) -> mean over each destination's
//   in-edges of msg (aggr_msg) and of x_rel*phi (x_update) -> x' = eta*x0 + (1-eta)*x + x_update.
// The first Linear of the edge MLP is split: its [h_src | h_dst] columns were applied per NODE
// by the projection stage (Psrc, Pdst(+bias)); only the 27+15 per-edge columns are a GEMM here.
// Per-edge activations never leave the SM.
#include "common.cuh"
#include "philox.cuh"

namespace eqd {

#define EDGE_K1 44    // 27 he + 15 rbf + 2 zero
#define EDGE_LD1 48   // smem row stride of the [he|rbf] operand
#define EDGE_LD 68    // smem row stride of 64-wide operands

struct EdgeSmem {
  float w1[EDGE_K1 * 64];
  float w2[64 * 64];
  float w3[64 * 64];
  float ln_g[64], ln_b[64], b2[64], b3[64], w4[64];
  float buf[EQD_TM * EDGE_LD];
  double xrel[EQD_TM * 3];
  float phi[EQD_TM];
  int src[EQD_TM];
  int dst[EQD_TM];
  int rp[EQD_TM + 1];
};

// DROP: training-mode dropout sites 0 (z1) and 1 (z3) of eqd_dropout `dr`, applied before their LeakyReLU.
template <bool DROP>
__global__ void __launch_bounds__(EQD_THREADS, 2)
edge_stage_kernel(eqd_graph g, eqd_layer_params p, const float* __restrict__ proj, const double* __restrict__ x_in,
                  const double* __restrict__ x_orig, float* __restrict__ aggr, double* __restrict__ x_out,
                  int* __restrict__ status, int tn /* destination nodes per tile */, eqd_dropout dr) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  EdgeSmem& s = *reinterpret_cast<EdgeSmem*>(smem_raw);
  const int tid = threadIdx.x, ty = tid >> 3, tx = tid & 7;
  const int pw = 128 + 3 * p.dhp;

  // layer weights -> shared memory, once per CTA
  for (int i = tid; i < EDGE_K1 * 64 / 4; i += EQD_THREADS)
    reinterpret_cast<float4*>(s.w1)[i] = reinterpret_cast<const float4*>(p.w_edge1)[i];
  for (int i = tid; i < 64 * 64 / 4; i += EQD_THREADS) {
    reinterpret_cast<float4*>(s.w2)[i] = reinterpret_cast<const float4*>(p.w_edge2)[i];
    reinterpret_cast<float4*>(s.w3)[i] = reinterpret_cast<const float4*>(p.w_coor1)[i];
  }
  if (tid < 64) {
    s.ln_g[tid] = p.edge_ln_g[tid];
    s.ln_b[tid] = p.edge_ln_b[tid];
    s.b2[tid] = p.b_edge2[tid];
    s.b3[tid] = p.b_coor1[tid];
    s.w4[tid] = p.w_coor2[tid];
  }
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

    // ---- per-edge geometry: thread t <-> edge e0+t ------------------------------------------
    {
      float* row = s.buf + tid * EDGE_LD1;
      if (tid < ne) {
        int e = e0 + tid;
        int sn = g.col_src[e], dn = g.edge_dst[e];
        s.src[tid] = sn;
        s.dst[tid] = dn;
        double rx = x_in[(long)sn * 3 + 0] - x_in[(long)dn * 3 + 0];  // u_sub_v :204-205
        double ry = x_in[(long)sn * 3 + 1] - x_in[(long)dn * 3 + 1];
        double rz = x_in[(long)sn * 3 + 2] - x_in[(long)dn * 3 + 2];
        s.xrel[tid * 3 + 0] = rx;
        s.xrel[tid * 3 + 1] = ry;
        s.xrel[tid * 3 + 2] = rz;
        float d2 = (float)(rx * rx + ry * ry + rz * rz);  // :208-209
        float sigma = 1.f;
#pragma unroll
        for (int q = 0; q < EQD_N_RBF; ++q) {  // exp(-d^2 / 1.5^q) :210
          row[EQD_EDGE_FEATS + q] = expf(-d2 / sigma);
          sigma *= 1.5f;
        }
      } else {
        s.src[tid] = -1;
        s.dst[tid] = -1;
#pragma unroll
        for (int q = 0; q < EQD_N_RBF; ++q) row[EQD_EDGE_FEATS + q] = 0.f;
      }
      row[42] = 0.f;
      row[43] = 0.f;
    }
    // original edge features he (E,27): the tile's rows are contiguous in one of the two arrays
    for (int idx = tid; idx < EQD_TM * EQD_EDGE_FEATS; idx += EQD_THREADS) {
      int r = idx / EQD_EDGE_FEATS, k = idx - r * EQD_EDGE_FEATS;
      float v = 0.f;
      if (r < ne) {
        int e = e0 + r;
        v = e < g.n_lig_edges ? g.he_lig[(long)e * EQD_EDGE_FEATS + k]
                              : g.he_rec[(long)(e - g.n_lig_edges) * EQD_EDGE_FEATS + k];
      }
      s.buf[r * EDGE_LD1 + k] = v;
    }
    __syncthreads();

    // ---- edge_mlp.0: gathered node projections + [he|rbf] GEMM -------------------------------
    float acc[8][8], accx[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      int r = ty * 8 + i;
      int sn = s.src[r], dn = s.dst[r];
      if (sn >= 0) {
        const float* ps = proj + (long)sn * pw + tx * 4;       // Psrc row
        const float* pd = proj + (long)dn * pw + 64 + tx * 4;  // Pdst row (+bias)
        float4 a0 = *reinterpret_cast<const float4*>(ps), a1 = *reinterpret_cast<const float4*>(ps + 32);
        float4 b0 = *reinterpret_cast<const float4*>(pd), b1 = *reinterpret_cast<const float4*>(pd + 32);
        acc[i][0] = a0.x + b0.x; acc[i][1] = a0.y + b0.y; acc[i][2] = a0.z + b0.z; acc[i][3] = a0.w + b0.w;
        acc[i][4] = a1.x + b1.x; acc[i][5] = a1.y + b1.y; acc[i][6] = a1.z + b1.z; acc[i][7] = a1.w + b1.w;
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
      }
    }
    gemm_nn<false>(acc, accx, s.buf + ty * 8 * EDGE_LD1, EDGE_LD1, s.w1, 64, EDGE_K1, tx);
    if (DROP) dropout_tile<false>(acc, accx, dr, 0, e0 + ty * 8, tx);
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

    // ---- coors_mlp: Linear, LeakyReLU, Linear(64->1) -> phi ------------------------------------
    acc_set_bias(acc, s.b3, tx);
    gemm_nn<false>(acc, accx, s.buf + ty * 8 * EDGE_LD, EDGE_LD, s.w3, 64, 64, tx);
    if (DROP) dropout_tile<false>(acc, accx, dr, 1, e0 + ty * 8, tx);
    {
      float w4r[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) w4r[j] = s.w4[col_nn(tx, j)];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float v = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) v = fmaf(lrelu(acc[i][j], p.leaky_slope), w4r[j], v);
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

}  // namespace eqd

extern "C" int eqd_edge_stage_ffma(const eqd_graph* g, const eqd_layer* p_l, const float* proj, const double* x_in,
                              const double* x_orig, float* aggr, double* x_out, int32_t* status, void* stream) {
  const eqd_layer_params* p = p_l ? &p_l->dev : nullptr;
  if (!g || !p || !proj || !x_in || !x_orig || !aggr || !x_out || !status) return EQD_ERR_BAD_ARG;
  if (g->max_in_degree < 1 || g->max_in_degree > EQD_TM) return EQD_ERR_UNSUPPORTED;
  if (!(p->leaky_slope >= 0.f && p->leaky_slope <= 1.f)) return EQD_ERR_UNSUPPORTED;  // lrelu() = max(v, slope*v)
  if (g->n_nodes <= 0) return EQD_OK;
  int tn = EQD_TM / g->max_in_degree;
  if (tn > EQD_TM) tn = EQD_TM;
  int ntiles = (g->n_nodes + tn - 1) / tn;
  size_t smem = sizeof(eqd::EdgeSmem);
  int grid = ntiles < EQD_SMS * 2 ? ntiles : EQD_SMS * 2;
  if (p_l->dropout.p > 0.f) {
    EQD_SET_SMEM((eqd::edge_stage_kernel<true>), smem);
    eqd::edge_stage_kernel<true><<<grid, EQD_THREADS, smem, (cudaStream_t)stream>>>(*g, *p, proj, x_in, x_orig, aggr,
                                                                                  x_out, status, tn, p_l->dropout);
  } else {
    EQD_SET_SMEM((eqd::edge_stage_kernel<false>), smem);
    eqd::edge_stage_kernel<false><<<grid, EQD_THREADS, smem, (cudaStream_t)stream>>>(*g, *p, proj, x_in, x_orig, aggr,
                                                                                   x_out, status, tn, p_l->dropout);
  }
  EQD_CUDA_LAUNCH_CHECK();
  return EQD_OK;
}
