// Node stage of IEGMN_Layer.forward (rigid_docking_model.py:244-256, 319-349), one fused kernel
// per layer.  A CTA owns a tile of <=128 nodes of ONE protein (segment) and
//   1. streams the partner protein's K / V rows (this layer's projections) through shared memory
//      and does flash-style cross attention  mu = softmax_j(q k_j^T) v_j  with an fp32 online
//      softmax -- the per-pair block of the reference's dense masked softmax (:61-63), no 1/sqrt(d);
//   2. node MLP on [h | aggr_msg | mu | h0] (Linear, LeakyReLU, LayerNorm, Linear) + skip (:332-337);
//   3. writes h' and, when a next layer exists, that layer's projections of h' (Psrc, Pdst, Q, K, V)
//      so h' is never re-read from HBM for them; with mu != NULL also mu (the per-layer backward reads it).
#include "common.cuh"
#include "philox.cuh"

namespace eqd {

template <bool EXTRA>
struct NodeCfg {
  static constexpr int DHP = EXTRA ? 72 : 64;
  // smem row stride of tiles: 68 for the 64-wide layers (conflict-free); the 72-wide layer 0 uses an unpadded 72
  // (2-way conflicts on the K-chunk reads of Q K^T only) so that two CTAs fit per SM (110.6 KB each)
  static constexpr int LD = EXTRA ? DHP : DHP + 4;
  static constexpr int KC = 64;       // keys per attention chunk
  static constexpr int BUF = EQD_TM * LD;
  static constexpr int KV = KC * LD + KC * DHP;  // K chunk (row stride LD) + V chunk (row stride DHP)
  static constexpr int WB = 2 * EQD_WCHUNK * EQD_WLD;
  static constexpr int KVW = KV > WB ? KV : WB;  // weight ring aliases the K/V staging area
  static constexpr size_t SMEM = (size_t)(2 * BUF + KVW) * sizeof(float);
};

// DROP: training-mode dropout site 2 (u5) of eqd_dropout `dr`, applied before the LeakyReLU.
template <bool EXTRA, bool DROP>
__global__ void __launch_bounds__(EQD_THREADS, 2)
node_stage_kernel(eqd_graph g, eqd_layer_params p, eqd_layer_params pn, int has_next, const float* __restrict__ h_in,
                  int ldh, const float* __restrict__ h0, const float* __restrict__ proj,
                  const float* __restrict__ aggr, float* __restrict__ h_out, float* __restrict__ proj_next,
                  float* __restrict__ mu_out, eqd_dropout dr) {
  using C = NodeCfg<EXTRA>;
  constexpr int DHP = C::DHP, LD = C::LD, KC = C::KC;
  extern __shared__ __align__(16) float smem[];
  float* bufA = smem;
  float* bufB = smem + C::BUF;
  float* Ks = smem + 2 * C::BUF;
  float* Vs = Ks + KC * LD;
  float* wbuf = Ks;  // alias: only used after the attention phase
  const int tid = threadIdx.x, ty = tid >> 3, tx = tid & 7;
  const int pw = 128 + 3 * DHP;
  const int B = g.n_pairs;

  for (int tile = blockIdx.x; tile < g.n_node_tiles; tile += gridDim.x) {
    const int seg = g.node_tiles[2 * tile], node0 = g.node_tiles[2 * tile + 1];
    const int nvalid = min(EQD_TM, g.seg_ptr[seg + 1] - node0);
    const int pseg = seg < B ? seg + B : seg - B;  // ligand <-> receptor of the same pair
    const int j0 = g.seg_ptr[pseg], j1 = g.seg_ptr[pseg + 1];

    // ================= cross attention (:247-256) =================
    tile_load_async(bufA, LD, proj + (long)node0 * pw + 128, pw, EQD_TM, nvalid, DHP, tid);  // Q tile
    cp_async_commit();
    float o[8][8], ox[8], m[8], l[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      m[i] = -INFINITY;
      l[i] = 0.f;
      ox[i] = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) o[i][j] = 0.f;
    }
    for (int jc = j0; jc < j1; jc += KC) {
      const int nk = min(KC, j1 - jc);
      tile_load_async(Ks, LD, proj + (long)jc * pw + 128 + DHP, pw, KC, nk, DHP, tid);
      tile_load_async(Vs, DHP, proj + (long)jc * pw + 128 + 2 * DHP, pw, KC, nk, DHP, tid);
      cp_async_commit();
      cp_async_wait<0>();
      __syncthreads();
      float s[8][8];
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) s[i][j] = 0.f;
      gemm_nt(s, bufA + ty * 8 * LD, LD, Ks, LD, DHP, tx);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float rmax = -INFINITY;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          if (col_nt(tx, j) >= nk) s[i][j] = -INFINITY;
          rmax = fmaxf(rmax, s[i][j]);
        }
        rmax = row_max8(rmax);
        float mnew = fmaxf(m[i], rmax);
        float scale = expf(m[i] - mnew);
        float rsum = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          float pj = expf(s[i][j] - mnew);
          s[i][j] = pj;
          rsum += pj;
        }
        rsum = row_sum8(rsum);
        l[i] = l[i] * scale + rsum;
        m[i] = mnew;
#pragma unroll
        for (int j = 0; j < 8; ++j) o[i][j] *= scale;
        if (EXTRA) ox[i] *= scale;
        float* pr = bufB + (ty * 8 + i) * LD + tx;
#pragma unroll
        for (int j = 0; j < 8; ++j) pr[8 * j] = s[i][j];
      }
      __syncthreads();
      gemm_nn<EXTRA>(o, ox, bufB + ty * 8 * LD, LD, Vs, DHP, KC, tx);
      __syncthreads();
    }
    // mu -> bufB (first operand of the node MLP)
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float inv = l[i] > 0.f ? 1.f / l[i] : 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) o[i][j] *= inv;
      if (EXTRA) ox[i] *= inv;
    }
    store_tile_smem<EXTRA>(bufB, LD, o, ox, ty, tx);
    if (mu_out) {  // mu[n][DHP]; columns 69..71 of the 72-wide layer are 0 (the padded V columns are 0)
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int r = ty * 8 + i;
        if (r < nvalid) {
          float* mrow = mu_out + (long)(node0 + r) * DHP;
          *reinterpret_cast<float4*>(mrow + tx * 4) = make_float4(o[i][0], o[i][1], o[i][2], o[i][3]);
          *reinterpret_cast<float4*>(mrow + 32 + tx * 4) = make_float4(o[i][4], o[i][5], o[i][6], o[i][7]);
          if (EXTRA) mrow[64 + tx] = ox[i];
        }
      }
    }

    // ================= node MLP (:319-337) =================
    const float* w5 = p.w_node1;  // [DHP + 64 + DHP + 72][DHP], row blocks [h | aggr | mu | h0]
    float acc[8][8], accx[8];
    acc_set_bias(acc, p.b_node1, tx);
#pragma unroll
    for (int i = 0; i < 8; ++i) accx[i] = EXTRA ? p.b_node1[64 + tx] : 0.f;
    tile_load_async(bufA, LD, h_in + (long)node0 * ldh, ldh, EQD_TM, nvalid, DHP, tid);  // h tile (Q is dead)
    cp_async_commit();
    cp_async_wait<0>();
    __syncthreads();
    gemm_nn_stream<EXTRA>(acc, accx, bufB + ty * 8 * LD, LD, DHP, w5 + (long)(DHP + 64) * DHP, DHP, DHP, wbuf, tid);
    gemm_nn_stream<EXTRA>(acc, accx, bufA + ty * 8 * LD, LD, DHP, w5, DHP, DHP, wbuf, tid);
    tile_load_async(bufB, LD, aggr + (long)node0 * 64, 64, EQD_TM, nvalid, 64, tid);
    tile_load_async(bufA, LD, h0 + (long)node0 * EQD_H0_PAD, EQD_H0_PAD, EQD_TM, nvalid, 64, tid);
    cp_async_commit();
    cp_async_wait<0>();
    __syncthreads();
    gemm_nn_stream<EXTRA>(acc, accx, bufB + ty * 8 * LD, LD, 64, w5 + (long)DHP * DHP, DHP, DHP, wbuf, tid);
    gemm_nn_stream<EXTRA>(acc, accx, bufA + ty * 8 * LD, LD, 64, w5 + (long)(2 * DHP + 64) * DHP, DHP, DHP, wbuf,
                          tid);
    tile_load_async(bufB, LD, h0 + (long)node0 * EQD_H0_PAD + 64, EQD_H0_PAD, EQD_TM, nvalid, 8, tid);
    cp_async_commit();
    cp_async_wait<0>();
    __syncthreads();
    gemm_nn_stream<EXTRA>(acc, accx, bufB + ty * 8 * LD, LD, 8, w5 + (long)(2 * DHP + 128) * DHP, DHP, DHP, wbuf,
                          tid);
    if (DROP) dropout_tile<EXTRA>(acc, accx, dr, 2, node0 + ty * 8, tx);
    lrelu_layernorm<EXTRA>(acc, accx, p.node_ln_g, p.node_ln_b, p.dh, p.leaky_slope, tx);
    store_tile_smem<EXTRA>(bufA, LD, acc, accx, ty, tx);
    __syncthreads();
    acc_set_bias(acc, p.b_node2, tx);
    gemm_nn_stream<false>(acc, accx, bufA + ty * 8 * LD, LD, DHP, p.w_node2, 64, 64, wbuf, tid);

    // skip connection (only when in/out widths match, :332-334), write h'
    const bool skip = (p.dh == EQD_HID);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      int r = ty * 8 + i;
      if (r < nvalid) {
        if (skip) {
          const float* hr = h_in + (long)(node0 + r) * ldh + tx * 4;
          float4 a = *reinterpret_cast<const float4*>(hr), b = *reinterpret_cast<const float4*>(hr + 32);
          const float sk = p.skip_weight_h, sk1 = 1.f - p.skip_weight_h;
          acc[i][0] = sk * acc[i][0] + sk1 * a.x; acc[i][1] = sk * acc[i][1] + sk1 * a.y;
          acc[i][2] = sk * acc[i][2] + sk1 * a.z; acc[i][3] = sk * acc[i][3] + sk1 * a.w;
          acc[i][4] = sk * acc[i][4] + sk1 * b.x; acc[i][5] = sk * acc[i][5] + sk1 * b.y;
          acc[i][6] = sk * acc[i][6] + sk1 * b.z; acc[i][7] = sk * acc[i][7] + sk1 * b.w;
        }
        float* orow = h_out + (long)(node0 + r) * EQD_HID + tx * 4;
        *reinterpret_cast<float4*>(orow) = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
        *reinterpret_cast<float4*>(orow + 32) = make_float4(acc[i][4], acc[i][5], acc[i][6], acc[i][7]);
      }
    }
    if (has_next) {  // fused projections of h' for the next layer
      store_tile_smem<false>(bufB, LD, acc, accx, ty, tx);
      __syncthreads();
      project_tile<false>(bufB, LD, pn, proj_next, node0, nvalid, wbuf, tid);
    }
    __syncthreads();
  }
}
}  // namespace eqd

extern "C" int eqd_node_stage(const eqd_graph* g, const eqd_layer* p_l, const eqd_layer* p_next_l, const float* h_in,
                              int32_t ldh, const float* h0, const float* proj, const float* aggr, float* mu,
                              float* h_out, float* proj_next, void* stream) {
  const eqd_layer_params* p = p_l ? &p_l->dev : nullptr;
  const eqd_layer_params* p_next = p_next_l ? &p_next_l->dev : nullptr;
  if (!g || !p || !h_in || !h0 || !proj || !aggr || !h_out) return EQD_ERR_BAD_ARG;
  if (reinterpret_cast<uintptr_t>(mu) & 15) return EQD_ERR_BAD_ARG;   // rows are written 16 bytes at a time
  if (p_next && (!proj_next || p_next->dh != 64 || p_next->dhp != 64)) return EQD_ERR_BAD_ARG;
  const bool extra = (p->dh == 69 && p->dhp == 72);
  if (!extra && !(p->dh == 64 && p->dhp == 64)) return EQD_ERR_UNSUPPORTED;
  if (!(p->leaky_slope >= 0.f && p->leaky_slope <= 1.f)) return EQD_ERR_UNSUPPORTED;  // lrelu() = max(v, slope*v)
  if (g->n_node_tiles <= 0) return EQD_OK;
  eqd_layer_params pn = p_next ? *p_next : *p;
  int has_next = p_next ? 1 : 0;
  cudaStream_t st = (cudaStream_t)stream;
  const eqd_dropout& dr = p_l->dropout;
  const int grid = g->n_node_tiles < EQD_SMS * 2 ? g->n_node_tiles : EQD_SMS * 2;
#define EQD_NODE_STAGE_LAUNCH(EXTRA, DROP)                                                                              \
  do {                                                                                                                \
    size_t smem = eqd::NodeCfg<EXTRA>::SMEM;                                                                          \
    EQD_SET_SMEM((eqd::node_stage_kernel<EXTRA, DROP>), smem);                                                        \
    eqd::node_stage_kernel<EXTRA, DROP><<<grid, EQD_THREADS, smem, st>>>(*g, *p, pn, has_next, h_in, ldh, h0, proj, aggr, \
                                                                         h_out, proj_next, mu, dr);                   \
  } while (0)
  if (dr.p > 0.f) {
    if (extra) EQD_NODE_STAGE_LAUNCH(true, true);
    else EQD_NODE_STAGE_LAUNCH(false, true);
  } else {
    if (extra) EQD_NODE_STAGE_LAUNCH(true, false);
    else EQD_NODE_STAGE_LAUNCH(false, false);
  }
#undef EQD_NODE_STAGE_LAUNCH
  EQD_CUDA_LAUNCH_CHECK();
  return EQD_OK;
}

extern "C" int eqd_iegmn_layer_forward(const eqd_graph* g, const eqd_layer* p_l, const eqd_layer* p_next_l,
                                       const float* h_in, int32_t ldh, const float* h0, const double* x_in,
                                       const double* x_orig, float* proj, float* proj_next, float* aggr, float* mu,
                                       float* h_out, double* x_out, int32_t* status, void* stream) {
  int rc = eqd_edge_stage(g, p_l, proj, x_in, x_orig, aggr, x_out, status, stream);
  if (rc) return rc;
  return eqd_node_stage(g, p_l, p_next_l, h_in, ldh, h0, proj, aggr, mu, h_out, proj_next, stream);
}
