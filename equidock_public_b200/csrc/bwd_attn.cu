// Backward of the segmented cross attention of IEGMN_Layer.forward (rigid_docking_model.py:46-64, 244-256):
//   mu_i = sum_j P_ij v_j,  P = softmax_j(q_i . k_j)  over the partner protein's nodes (no 1/sqrt(d)).
// Flash-attention style, two kernels, no atomics, nothing N x M ever stored:
//   bwd_attn_dq_kernel : tile = 128 query rows.  Pass 1 recomputes the row max / row sum over all key chunks; pass 2
//                        recomputes P chunk by chunk, dP = dmu . V^T, dS = P (dP - D), D_i = dmu_i . mu_i, dQ += dS . K.
//                        Writes dQ * lrelu'(Q) and the row statistics (m, l, D).
//   bwd_attn_dkv_kernel: tile = 128 key rows; loops over the partner's query chunks: P^T from the saved statistics,
//                        dV += P^T . dmu, dS^T = P^T (V . dmu^T - D), dK += dS^T . Q.  Writes dK * lrelu'(K) and dV.
// Gradients land in the combined projection-gradient matrix dP[n][128 + 3 dhp] = [dPsrc | dPdst | dQpre | dKpre | dV].
// Restated in oracle/backward_manual.py::attn_bwd.
#include "bwd_common.cuh"

namespace eqd {

template <bool EXTRA>
struct AttnBwdCfg {
  static constexpr int DHP = EXTRA ? 72 : 64;
  static constexpr int LD = DHP + 4;
  static constexpr int KC = 64;
  static constexpr int BUF = EQD_TM * LD;
  static constexpr int CH = KC * LD;
  static constexpr size_t SMEM_DQ = (size_t)(3 * BUF + 2 * CH) * sizeof(float);
  static constexpr size_t SMEM_DKV = (size_t)(4 * BUF + 2 * CH + 3 * KC) * sizeof(float);
};

template <bool EXTRA>
__global__ void __launch_bounds__(EQD_THREADS)
bwd_attn_dq_kernel(eqd_graph g, float slope, const float* __restrict__ proj, const float* __restrict__ mu, int ldmu,
                   const float* __restrict__ dmu, float* __restrict__ dP, float* __restrict__ rowstat /*[n][4]*/) {
  using C = AttnBwdCfg<EXTRA>;
  constexpr int DHP = C::DHP, LD = C::LD, KC = C::KC;
  extern __shared__ __align__(16) float smem[];
  float* bufQ = smem;
  float* bufD = smem + C::BUF;       // dmu tile
  float* bufS = smem + 2 * C::BUF;   // dS chunk (A operand of dQ += dS . K)
  float* Ks = smem + 3 * C::BUF;
  float* Vs = Ks + C::CH;
  const int tid = threadIdx.x, ty = tid >> 3, tx = tid & 7;
  const int pw = 128 + 3 * DHP, B = g.n_pairs;

  for (int tile = blockIdx.x; tile < g.n_node_tiles; tile += gridDim.x) {
    const int seg = g.node_tiles[2 * tile], node0 = g.node_tiles[2 * tile + 1];
    const int nvalid = min(EQD_TM, g.seg_ptr[seg + 1] - node0);
    const int pseg = seg < B ? seg + B : seg - B;
    const int j0 = g.seg_ptr[pseg], j1 = g.seg_ptr[pseg + 1];
    tile_load_async(bufQ, LD, proj + (long)node0 * pw + 128, pw, EQD_TM, nvalid, DHP, tid);
    tile_load_async(bufD, LD, dmu + (long)node0 * DHP, DHP, EQD_TM, nvalid, DHP, tid);
    cp_async_commit();
    // ---- pass 1: row max and row sum of exp over all keys ----
    float m[8], l[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) { m[i] = -INFINITY; l[i] = 0.f; }
    for (int jc = j0; jc < j1; jc += KC) {
      const int nk = min(KC, j1 - jc);
      tile_load_async(Ks, LD, proj + (long)jc * pw + 128 + DHP, pw, KC, nk, DHP, tid);
      cp_async_commit();
      cp_async_wait<0>();
      __syncthreads();
      float s[8][8];
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) s[i][j] = 0.f;
      gemm_nt(s, bufQ + ty * 8 * LD, LD, Ks, LD, DHP, tx);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float rmax = -INFINITY;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          if (col_nt(tx, j) >= nk) s[i][j] = -INFINITY;
          rmax = fmaxf(rmax, s[i][j]);
        }
        rmax = row_max8(rmax);
        const float mnew = fmaxf(m[i], rmax);
        float rsum = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) rsum += expf(s[i][j] - mnew);
        rsum = row_sum8(rsum);
        l[i] = l[i] * expf(m[i] - mnew) + rsum;
        m[i] = mnew;
      }
      __syncthreads();
    }
    cp_async_wait<0>();
    __syncthreads();
    // ---- D_i = dmu_i . mu_i ----
    float Drow[8], linv[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int r = ty * 8 + i;
      float t = 0.f;
      if (r < nvalid) {
        const float* mr = mu + (long)(node0 + r) * ldmu;
        const float* dr = bufD + r * LD;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int c = col_nn(tx, j);
          t = fmaf(mr[c], dr[c], t);
        }
        if (EXTRA) t = fmaf(mr[64 + tx], dr[64 + tx], t);
      }
      Drow[i] = row_sum8(t);
      linv[i] = l[i] > 0.f ? 1.f / l[i] : 0.f;
      if (tx == 0 && r < nvalid) {
        float* rs = rowstat + (long)(node0 + r) * 4;
        rs[0] = m[i]; rs[1] = linv[i]; rs[2] = Drow[i]; rs[3] = 0.f;
      }
    }
    // ---- pass 2: dQ ----
    float o[8][8], ox[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      ox[i] = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) o[i][j] = 0.f;
    }
    for (int jc = j0; jc < j1; jc += KC) {
      const int nk = min(KC, j1 - jc);
      tile_load_async(Ks, LD, proj + (long)jc * pw + 128 + DHP, pw, KC, nk, DHP, tid);
      tile_load_async(Vs, LD, proj + (long)jc * pw + 128 + 2 * DHP, pw, KC, nk, DHP, tid);
      cp_async_commit();
      cp_async_wait<0>();
      __syncthreads();
      float s[8][8], dp[8][8];
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) { s[i][j] = 0.f; dp[i][j] = 0.f; }
      gemm_nt(s, bufQ + ty * 8 * LD, LD, Ks, LD, DHP, tx);
      gemm_nt(dp, bufD + ty * 8 * LD, LD, Vs, LD, DHP, tx);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float* pr = bufS + (ty * 8 + i) * LD + tx;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float pj = col_nt(tx, j) < nk ? expf(s[i][j] - m[i]) * linv[i] : 0.f;
          pr[8 * j] = pj * (dp[i][j] - Drow[i]);
        }
      }
      __syncthreads();
      gemm_nn<EXTRA>(o, ox, bufS + ty * 8 * LD, LD, Ks, LD, KC, tx);
      __syncthreads();
    }
    // ---- dQpre = dQ * lrelu'(Q) -> dP[:, 128 : 128 + dhp] ----
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int r = ty * 8 + i;
      if (r < nvalid) {
        const float* qr = bufQ + r * LD;
        float v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = o[i][j] * lrelu_grad_from_post(qr[col_nn(tx, j)], slope);
        float* d = dP + (long)(node0 + r) * pw + 128 + tx * 4;
        *reinterpret_cast<float4*>(d) = make_float4(v[0], v[1], v[2], v[3]);
        *reinterpret_cast<float4*>(d + 32) = make_float4(v[4], v[5], v[6], v[7]);
        if (EXTRA) dP[(long)(node0 + r) * pw + 128 + 64 + tx] = ox[i] * lrelu_grad_from_post(qr[64 + tx], slope);
      }
    }
    __syncthreads();
  }
}

template <bool EXTRA>
__global__ void __launch_bounds__(EQD_THREADS)
bwd_attn_dkv_kernel(eqd_graph g, float slope, const float* __restrict__ proj, const float* __restrict__ dmu,
                    const float* __restrict__ rowstat, float* __restrict__ dP) {
  using C = AttnBwdCfg<EXTRA>;
  constexpr int DHP = C::DHP, LD = C::LD, KC = C::KC;
  extern __shared__ __align__(16) float smem[];
  float* bufK = smem;
  float* bufV = smem + C::BUF;
  float* bufP = smem + 2 * C::BUF;   // P^T chunk
  float* bufS = smem + 3 * C::BUF;   // dS^T chunk
  float* Qc = smem + 4 * C::BUF;     // [64][LD]
  float* Dc = Qc + C::CH;            // dmu chunk [64][LD]
  float* st = Dc + C::CH;            // [3][64]: m, 1/l, D of the chunk's query rows
  const int tid = threadIdx.x, ty = tid >> 3, tx = tid & 7;
  const int pw = 128 + 3 * DHP, B = g.n_pairs;

  for (int tile = blockIdx.x; tile < g.n_node_tiles; tile += gridDim.x) {
    const int seg = g.node_tiles[2 * tile], node0 = g.node_tiles[2 * tile + 1];
    const int nvalid = min(EQD_TM, g.seg_ptr[seg + 1] - node0);
    const int pseg = seg < B ? seg + B : seg - B;           // the queries that attend to these keys
    const int i0 = g.seg_ptr[pseg], i1 = g.seg_ptr[pseg + 1];
    tile_load_async(bufK, LD, proj + (long)node0 * pw + 128 + DHP, pw, EQD_TM, nvalid, DHP, tid);
    tile_load_async(bufV, LD, proj + (long)node0 * pw + 128 + 2 * DHP, pw, EQD_TM, nvalid, DHP, tid);
    cp_async_commit();
    float ok[8][8], okx[8], ov[8][8], ovx[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      okx[i] = ovx[i] = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) ok[i][j] = ov[i][j] = 0.f;
    }
    for (int ic = i0; ic < i1; ic += KC) {
      const int nq = min(KC, i1 - ic);
      tile_load_async(Qc, LD, proj + (long)ic * pw + 128, pw, KC, nq, DHP, tid);
      tile_load_async(Dc, LD, dmu + (long)ic * DHP, DHP, KC, nq, DHP, tid);
      cp_async_commit();
      if (tid < KC) {
        const bool okq = tid < nq;
        const float* rs = rowstat + (long)(ic + (okq ? tid : 0)) * 4;
        st[tid] = okq ? rs[0] : 0.f;
        st[KC + tid] = okq ? rs[1] : 0.f;
        st[2 * KC + tid] = okq ? rs[2] : 0.f;
      }
      cp_async_wait<0>();
      __syncthreads();
      float s[8][8], dp[8][8];
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) { s[i][j] = 0.f; dp[i][j] = 0.f; }
      gemm_nt(s, bufK + ty * 8 * LD, LD, Qc, LD, DHP, tx);     // S^T[key][query]
      gemm_nt(dp, bufV + ty * 8 * LD, LD, Dc, LD, DHP, tx);    // dP^T[key][query] = v_key . dmu_query
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int c = col_nt(tx, j);
        const bool okc = c < nq;
        const float mq = st[c], liq = st[KC + c], dq = st[2 * KC + c];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float pt = okc ? expf(s[i][j] - mq) * liq : 0.f;
          bufP[(ty * 8 + i) * LD + c] = pt;
          bufS[(ty * 8 + i) * LD + c] = pt * (dp[i][j] - dq);
        }
      }
      __syncthreads();
      gemm_nn<EXTRA>(ov, ovx, bufP + ty * 8 * LD, LD, Dc, LD, KC, tx);   // dV += P^T . dmu
      gemm_nn<EXTRA>(ok, okx, bufS + ty * 8 * LD, LD, Qc, LD, KC, tx);   // dK += dS^T . Q
      __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int r = ty * 8 + i;
      if (r < nvalid) {
        const float* kr = bufK + r * LD;
        float v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = ok[i][j] * lrelu_grad_from_post(kr[col_nn(tx, j)], slope);
        float* d = dP + (long)(node0 + r) * pw + 128 + DHP + tx * 4;
        *reinterpret_cast<float4*>(d) = make_float4(v[0], v[1], v[2], v[3]);
        *reinterpret_cast<float4*>(d + 32) = make_float4(v[4], v[5], v[6], v[7]);
        float* e = dP + (long)(node0 + r) * pw + 128 + 2 * DHP + tx * 4;
        *reinterpret_cast<float4*>(e) = make_float4(ov[i][0], ov[i][1], ov[i][2], ov[i][3]);
        *reinterpret_cast<float4*>(e + 32) = make_float4(ov[i][4], ov[i][5], ov[i][6], ov[i][7]);
        if (EXTRA) {
          dP[(long)(node0 + r) * pw + 128 + DHP + 64 + tx] = okx[i] * lrelu_grad_from_post(kr[64 + tx], slope);
          dP[(long)(node0 + r) * pw + 128 + 2 * DHP + 64 + tx] = ovx[i];
        }
      }
    }
    __syncthreads();
  }
}

}  // namespace eqd

extern "C" int eqd_bwd_attention(const eqd_graph* g, const eqd_layer* p_l, const float* proj, const float* mu,
                                 int32_t ldmu, const float* dmu, float* dP, float* rowstat, void* stream) {
  const eqd_layer_params* p = p_l ? &p_l->dev : nullptr;
  if (!g || !p || !proj || !mu || !dmu || !dP || !rowstat) return EQD_ERR_BAD_ARG;
  const bool extra = (p->dh == 69 && p->dhp == 72);
  if (!extra && !(p->dh == 64 && p->dhp == 64)) return EQD_ERR_UNSUPPORTED;
  if (!(p->leaky_slope >= 0.f && p->leaky_slope <= 1.f)) return EQD_ERR_UNSUPPORTED;
  if (g->n_node_tiles <= 0) return EQD_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = g->n_node_tiles < EQD_SMS ? g->n_node_tiles : EQD_SMS;
  if (extra) {
    EQD_SET_SMEM((eqd::bwd_attn_dq_kernel<true>), eqd::AttnBwdCfg<true>::SMEM_DQ);
    eqd::bwd_attn_dq_kernel<true><<<grid, EQD_THREADS, eqd::AttnBwdCfg<true>::SMEM_DQ, st>>>(*g, p->leaky_slope, proj, mu,
                                                                                            ldmu, dmu, dP, rowstat);
    EQD_CUDA_LAUNCH_CHECK();
    EQD_SET_SMEM((eqd::bwd_attn_dkv_kernel<true>), eqd::AttnBwdCfg<true>::SMEM_DKV);
    eqd::bwd_attn_dkv_kernel<true><<<grid, EQD_THREADS, eqd::AttnBwdCfg<true>::SMEM_DKV, st>>>(*g, p->leaky_slope, proj, dmu,
                                                                                              rowstat, dP);
  } else {
    EQD_SET_SMEM((eqd::bwd_attn_dq_kernel<false>), eqd::AttnBwdCfg<false>::SMEM_DQ);
    eqd::bwd_attn_dq_kernel<false><<<grid, EQD_THREADS, eqd::AttnBwdCfg<false>::SMEM_DQ, st>>>(*g, p->leaky_slope, proj, mu,
                                                                                              ldmu, dmu, dP, rowstat);
    EQD_CUDA_LAUNCH_CHECK();
    EQD_SET_SMEM((eqd::bwd_attn_dkv_kernel<false>), eqd::AttnBwdCfg<false>::SMEM_DKV);
    eqd::bwd_attn_dkv_kernel<false><<<grid, EQD_THREADS, eqd::AttnBwdCfg<false>::SMEM_DKV, st>>>(*g, p->leaky_slope, proj,
                                                                                                dmu, rowstat, dP);
  }
  EQD_CUDA_LAUNCH_CHECK();
  return EQD_OK;
}
