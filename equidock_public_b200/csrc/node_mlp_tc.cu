// Node MLP of a 64-wide IEGMN layer (rigid_docking_model.py:319-337) on the tensor cores (wgmma, bf16x6):
//   h' = skip( W6 . LayerNorm(LeakyReLU(W5 . [h | aggr_msg | mu | h0] + b5)) + b6 )
// Weight-stationary (W5: 64x272, W6: 64x64 as bf16x3 panels, 126 KB in shared memory); one tile of 128 node rows per
// CTA of 256 threads at a time (2 threads per node row, two 64-row warpgroup slabs in the GEMMs).  The 272-wide input
// is fed in 5 K-pieces; the A operand region takes each piece's fp32 result tile once its MMAs are complete.
#include "tc_common.cuh"

namespace eqd {

#define NM_THREADS 256
#define NM_W5_SPLIT 34816   // 64 x 272 bf16
#define NM_W6_BASE 104448
#define NM_W6_SPLIT 8192
#define NM_W_BYTES 129024
#define NM_A_SPLIT 16384    // A operand: 128 rows x 64 bf16 per split
#define NM_LD 68            // fp32 row stride of the result tile

struct NmConsts { float b5[64], ln_g[64], ln_b[64], b6[64]; };

#define NM_SC_LD 36   // padded row stride (floats) of a warp's 32 x 32 transposition scratch: conflict-free both ways

struct NmSmem {
  unsigned char w[NM_W_BYTES];
  unsigned char a[3 * NM_A_SPLIT];
  float sc[NM_THREADS / 32][32 * NM_SC_LD];   // one 32-row x 128-byte scratch per warp (its rows x its column half)
  float red[EQD_TM * 4];
  unsigned long long w_bar;
};

__global__ void __launch_bounds__(NM_THREADS, 1)
node_mlp_tc_kernel(int n_nodes, eqd_layer_params p, const __grid_constant__ NmConsts cst, const float* __restrict__ h_in,
                   const float* __restrict__ aggr, const float* __restrict__ mu, const float* __restrict__ h0,
                   float* __restrict__ h_out) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  NmSmem& S = *reinterpret_cast<NmSmem*>(smem_raw);
  const int tid = threadIdx.x, q = tid, half = q >> 7, r = q & 127, warp = tid >> 5, wgi = tid >> 7;
  const int ntiles = (n_nodes + EQD_TM - 1) / EQD_TM;
  TRACE_START(3);
  if (tid == 0) {
    mbar_init(&S.w_bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    mbar_expect_tx(&S.w_bar, NM_W_BYTES);
    bulk_g2s(S.w, p.w_node_tc, NM_W_BYTES, &S.w_bar);
  }
  __syncthreads();
  const unsigned w_saddr = smem_u32(S.w), a_saddr = smem_u32(S.a);
  float* const dtile = reinterpret_cast<float*>(S.a);
  auto a_desc = [&](int sp, int kb) { return a_desc_at<EQD_TM>(a_saddr, NM_A_SPLIT, wgi, sp, kb); };
  mbar_wait(&S.w_bar, 0);
  const float slope = p.leaky_slope;
  float* red = S.red;

  // The A operand in place (callers fence + barrier first) times K-blocks [0, nkb) of the panel at w_off -> out (my row
  // half of the fresh product); on return the A region is free again.
  auto gemm = [&](unsigned w_off, unsigned w_split, int nkb, float (&out)[32]) {
    {
      float d[32];
      wg_gemm6<64>(d, a_desc, [&](int sp, int kb) { return b_desc_ex(w_saddr + w_off + sp * w_split + kb * 2048, 1024, 128); },
                   nkb, false);
      __syncthreads();
      wg_store_d<64>(dtile + wgi * 64 * NM_LD, NM_LD, d, tid & 127);
    }
    __syncthreads();
    tile_ld32f(dtile, NM_LD, r, half * 32, out);
    __syncthreads();
  };

  // Global rows travel coalesced: the warp's 32 rows x 128 bytes (its column half) are cp.async'ed into its scratch,
  // 8 lanes per row, one piece ahead of its use; each thread then picks up its own row.
  const int lane = tid & 31, wrow0 = 32 * (warp & 3);
  float* sc = S.sc[warp];
  auto fetch = [&](const float* base, int ld, int t) {
    if (t >= ntiles) return;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int row = i * 4 + (lane >> 3);
      const long nd = (long)t * EQD_TM + wrow0 + row;
      const bool ok = nd < n_nodes;   // src-size 0 zero-fills
      cp_async16(sc + row * NM_SC_LD + (lane & 7) * 4, base + (ok ? nd : 0) * ld + half * 32 + (lane & 7) * 4, ok);
    }
    cp_async_commit();
  };
  auto take = [&](float (&v)[32]) {
    cp_async_wait<0>();
    __syncwarp();
#pragma unroll
    for (int c4 = 0; c4 < 8; ++c4) {
      float4 t = *reinterpret_cast<const float4*>(sc + lane * NM_SC_LD + c4 * 4);
      v[c4 * 4] = t.x; v[c4 * 4 + 1] = t.y; v[c4 * 4 + 2] = t.z; v[c4 * 4 + 3] = t.w;
    }
    __syncwarp();
  };
  fetch(h_in, EQD_HID, blockIdx.x);
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    if (q == 0) TRACE_PHASE(3, blockIdx.x, tile, 1);
    const int node = tile * EQD_TM + r;
    const bool valid = node < n_nodes;
    // ---- node_mlp.0 over [h | aggr | mu | h0] in 5 K-pieces ---------------------------------------------------
    // Each 64-wide piece is its own accumulation (4 full-magnitude steps, like the edge-stage GEMMs) and the pieces
    // are summed in registers with round-to-nearest FADDs.
    float acc[32];
#pragma unroll
    for (int c = 0; c < 32; ++c) acc[c] = cst.b5[half * 32 + c];
    {
      float v[32], d[32];
      auto piece = [&](unsigned w_off, int nkb) {
        tc_fence_before();
        __syncthreads();
        gemm(w_off, NM_W5_SPLIT, nkb, d);
#pragma unroll
        for (int c = 0; c < 32; ++c) acc[c] += d[c];
      };
      take(v);
      fetch(aggr, EQD_HID, tile);
      store_half_split3<EQD_TM>(S.a, NM_A_SPLIT, r, half * 32, v);   // piece 0 (h) -> A
      piece(0, 4);
      take(v);
      fetch(mu, EQD_HID, tile);
      store_half_split3<EQD_TM>(S.a, NM_A_SPLIT, r, half * 32, v);   // piece 1 (aggr)
      piece(4 * 2048, 4);
      take(v);
      fetch(h0, EQD_H0_PAD, tile);
      store_half_split3<EQD_TM>(S.a, NM_A_SPLIT, r, half * 32, v);   // piece 2 (mu)
      piece(8 * 2048, 4);
      take(v);
      store_half_split3<EQD_TM>(S.a, NM_A_SPLIT, r, half * 32, v);   // piece 3 (h0[0:64])
      piece(12 * 2048, 4);
      // piece 4: h0[64:72] + 8 zero columns (K = 16): the half-0 threads write the k-block
      if (half == 0) {
        const float4* sp = reinterpret_cast<const float4*>(h0 + (long)node * EQD_H0_PAD + 64);
        float4 a = valid ? sp[0] : make_float4(0.f, 0.f, 0.f, 0.f), b = valid ? sp[1] : make_float4(0.f, 0.f, 0.f, 0.f);
        float t[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
        store_extra8_split3<EQD_TM>(S.a, NM_A_SPLIT, r, 0, t);
      }
      piece(16 * 2048, 1);
    }
    // ---- + bias, LeakyReLU, LayerNorm -> bf16x3 -> A ; node_mlp.4 ---------------------------------------------
    {
      float v[32];
      float s4[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int c = 0; c < 32; ++c) {
        v[c] = lrelu(acc[c], slope);
        s4[c & 3] += v[c];
      }
      const float mh = ((s4[0] + s4[1]) + (s4[2] + s4[3])) * (1.f / 32.f);
      float q4[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int c = 0; c < 32; ++c) {
        float d = v[c] - mh;
        q4[c & 3] = fmaf(d, d, q4[c & 3]);
      }
      red[(r * 2 + half) * 2 + 0] = mh;
      red[(r * 2 + half) * 2 + 1] = (q4[0] + q4[1]) + (q4[2] + q4[3]);
      __syncthreads();
      const float m0 = red[r * 4 + 0], m1 = red[r * 4 + 2];
      const float mean = 0.5f * (m0 + m1);
      const float dm = m0 - m1;
      const float var = (red[r * 4 + 1] + red[r * 4 + 3] + dm * dm * 16.f) * (1.f / 64.f);  // Chan et al. combination
      const float rstd = 1.f / sqrtf(var + 1e-5f);
#pragma unroll
      for (int c = 0; c < 32; ++c) v[c] = (v[c] - mean) * rstd * cst.ln_g[half * 32 + c] + cst.ln_b[half * 32 + c];
      store_half_split3<EQD_TM>(S.a, NM_A_SPLIT, r, half * 32, v);
    }
    fetch(h_in, EQD_HID, tile);   // the skip operand again (an L2 hit) rather than 32 registers held across the tile
    tc_fence_before();
    __syncthreads();
    {
      float v[32], hskip[32];
      gemm(NM_W6_BASE, NM_W6_SPLIT, 4, v);
      take(hskip);
      const float sk = p.skip_weight_h, sk1 = 1.f - p.skip_weight_h;
#pragma unroll
      for (int c = 0; c < 32; ++c) v[c] = sk * (v[c] + cst.b6[half * 32 + c]) + sk1 * hskip[c];  // :332-334
      // transposed through the scratch: 8 lanes write one contiguous 128-byte half row
#pragma unroll
      for (int c4 = 0; c4 < 8; ++c4)
        *reinterpret_cast<float4*>(sc + lane * NM_SC_LD + c4 * 4) = make_float4(v[c4 * 4], v[c4 * 4 + 1], v[c4 * 4 + 2], v[c4 * 4 + 3]);
      __syncwarp();
      float* o = h_out + ((long)tile * EQD_TM + wrow0) * EQD_HID + half * 32 + (lane & 7) * 4;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int row = i * 4 + (lane >> 3);
        float4 t = *reinterpret_cast<const float4*>(sc + row * NM_SC_LD + (lane & 7) * 4);
        if ((long)tile * EQD_TM + wrow0 + row < n_nodes) *reinterpret_cast<float4*>(o + (long)row * EQD_HID) = t;
      }
      __syncwarp();
    }
    fetch(h_in, EQD_HID, tile + gridDim.x);   // next tile's h rows
  }
  TRACE_END(3);
}


// ---- the 69-wide layer 0 ------------------------------------------------------------------------------------------------
// h = h0 here, so the h and h0 blocks of node_mlp.0 fold into one: hidden = W5' [h0 (69 -> 80) | aggr (64) | mu (69 -> 80)]
// with N = 69 -> 80 outputs; LayerNorm over the 69 real channels; node_mlp.4 as [64][80]; no skip (widths differ, :332).
// Column ownership of the 80-wide rows: half 0 = [0,32) and the extra [64,80), half 1 = [32,64).
#define NM0_W5_SPLIT 35840    // 80 x 224 bf16
#define NM0_W6_BASE 107520
#define NM0_W6_SPLIT 10240    // 64 x 80 bf16
#define NM0_W_BYTES 138240
#define NM0_A_SPLIT 20480     // A operand: 128 rows x 80 bf16 per split
#define NM0_LD 84             // fp32 row stride of the result tile

struct Nm0Consts { float b5[80], ln_g[80], ln_b[80], b6[64]; };

struct Nm0Smem {
  unsigned char w[NM0_W_BYTES];
  unsigned char a[3 * NM0_A_SPLIT];
  float red[EQD_TM * 4];
  unsigned long long w_bar;
};

__global__ void __launch_bounds__(NM_THREADS, 1)
node_mlp0_tc_kernel(int n_nodes, eqd_layer_params p, const __grid_constant__ Nm0Consts cst, const float* __restrict__ h0,
                    const float* __restrict__ aggr, const float* __restrict__ mu /*[n][72]*/, float* __restrict__ h_out) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  Nm0Smem& S = *reinterpret_cast<Nm0Smem*>(smem_raw);
  const int tid = threadIdx.x, q = tid, half = q >> 7, r = q & 127, wgi = tid >> 7;
  const int ntiles = (n_nodes + EQD_TM - 1) / EQD_TM;
  TRACE_START(3);
  if (tid == 0) {
    mbar_init(&S.w_bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    mbar_expect_tx(&S.w_bar, NM0_W_BYTES);
    bulk_g2s(S.w, p.w_node_tc, NM0_W_BYTES, &S.w_bar);
  }
  __syncthreads();
  const unsigned w_saddr = smem_u32(S.w), a_saddr = smem_u32(S.a);
  float* const dtile = reinterpret_cast<float*>(S.a);
  auto a_desc = [&](int sp, int kb) { return a_desc_at<EQD_TM>(a_saddr, NM0_A_SPLIT, wgi, sp, kb); };
  mbar_wait(&S.w_bar, 0);
  const float slope = p.leaky_slope;
  float* red = S.red;

  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    if (q == 0) TRACE_PHASE(3, blockIdx.x, tile, 1);
    const int node = tile * EQD_TM + r;
    const bool valid = node < n_nodes;
    auto row32 = [&](const float* base, int ld, float (&v)[32]) {   // my half row of a [n][ld] array
      const float4* sp = reinterpret_cast<const float4*>(base + (long)node * ld + half * 32);
#pragma unroll
      for (int c4 = 0; c4 < 8; ++c4) {
        float4 t = valid ? sp[c4] : make_float4(0.f, 0.f, 0.f, 0.f);
        v[c4 * 4] = t.x; v[c4 * 4 + 1] = t.y; v[c4 * 4 + 2] = t.z; v[c4 * 4 + 3] = t.w;
      }
    };
    // channels [64, 72) of an 72-strided row (zero beyond 69) as the piece's fifth k-block; half-0 threads only
    auto extra8 = [&](const float* base) {
      if (half == 0) {
        const float4* ep = reinterpret_cast<const float4*>(base + (long)node * EQD_H0_PAD + 64);
        float4 a = valid ? ep[0] : make_float4(0.f, 0.f, 0.f, 0.f), b = valid ? ep[1] : make_float4(0.f, 0.f, 0.f, 0.f);
        float t[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
        store_extra8_split3<EQD_TM>(S.a, NM0_A_SPLIT, r, 64, t);
      }
    };
    float acc[32], accx[16];   // accx: columns 64..79 (half 0)
#pragma unroll
    for (int c = 0; c < 32; ++c) acc[c] = cst.b5[half * 32 + c];
#pragma unroll
    for (int c = 0; c < 16; ++c) accx[c] = cst.b5[64 + c];
    // k-blocks [kb0, kb0 + nkb) of W5' against the A operand, a fresh accumulation summed here with RN adds (<= 5
    // full-magnitude steps each); on return the A region is free again
    auto piece = [&](int kb0, int nkb) {
      tc_fence_before();
      __syncthreads();
      {
        float d[40];
        wg_gemm6<80>(d, a_desc, [&](int sp, int kb) {
          return b_desc_ex(w_saddr + (kb0 + kb) * (80 * 32) + sp * NM0_W5_SPLIT, 80 * 16, 128); }, nkb, false);
        __syncthreads();
        wg_store_d<80>(dtile + wgi * 64 * NM0_LD, NM0_LD, d, tid & 127);
      }
      __syncthreads();
      const float* dr = dtile + r * NM0_LD;
#pragma unroll
      for (int c = 0; c < 32; ++c) acc[c] += dr[half * 32 + c];
      if (half == 0) {
#pragma unroll
        for (int c = 0; c < 16; ++c) accx[c] += dr[64 + c];
      }
      __syncthreads();
    };
    {
      float v[32];
      row32(h0, EQD_H0_PAD, v);
      store_half_split3<EQD_TM>(S.a, NM0_A_SPLIT, r, half * 32, v);   // piece 0: h0 (80)
      extra8(h0);
      piece(0, 5);
      row32(aggr, EQD_HID, v);
      store_half_split3<EQD_TM>(S.a, NM0_A_SPLIT, r, half * 32, v);   // piece 1: aggr (64)
      piece(5, 4);
      row32(mu, EQD_H0_PAD, v);
      store_half_split3<EQD_TM>(S.a, NM0_A_SPLIT, r, half * 32, v);   // piece 2: mu (80)
      extra8(mu);
      piece(9, 5);
    }
    // ---- LeakyReLU, LayerNorm over the 69 real channels -> bf16x3 -> A ; node_mlp.4 ---------------------------------
    {
      const int nh = half == 0 ? 37 : 32;
      float sum = 0.f;
#pragma unroll
      for (int c = 0; c < 32; ++c) {
        acc[c] = lrelu(acc[c], slope);
        sum += acc[c];
      }
      if (half == 0) {
#pragma unroll
        for (int c = 0; c < 5; ++c) {
          accx[c] = lrelu(accx[c], slope);
          sum += accx[c];
        }
      }
      const float mh = sum / (float)nh;
      float m2 = 0.f;
#pragma unroll
      for (int c = 0; c < 32; ++c) {
        float d = acc[c] - mh;
        m2 = fmaf(d, d, m2);
      }
      if (half == 0) {
#pragma unroll
        for (int c = 0; c < 5; ++c) {
          float d = accx[c] - mh;
          m2 = fmaf(d, d, m2);
        }
      }
      red[(r * 2 + half) * 2 + 0] = mh;
      red[(r * 2 + half) * 2 + 1] = m2;
      __syncthreads();
      const float m0 = red[r * 4 + 0], m1 = red[r * 4 + 2];
      const float mean = (37.f * m0 + 32.f * m1) * (1.f / 69.f);
      const float dm = m0 - m1;
      const float var = (red[r * 4 + 1] + red[r * 4 + 3] + dm * dm * (37.f * 32.f / 69.f)) * (1.f / 69.f);  // Chan et al.
      const float rstd = 1.f / sqrtf(var + 1e-5f);
#pragma unroll
      for (int c = 0; c < 32; ++c) acc[c] = (acc[c] - mean) * rstd * cst.ln_g[half * 32 + c] + cst.ln_b[half * 32 + c];
      store_half_split3<EQD_TM>(S.a, NM0_A_SPLIT, r, half * 32, acc);
      if (half == 0) {
        float t[8];
#pragma unroll
        for (int c = 0; c < 5; ++c) t[c] = (accx[c] - mean) * rstd * cst.ln_g[64 + c] + cst.ln_b[64 + c];
        t[5] = t[6] = t[7] = 0.f;
        store_extra8_split3<EQD_TM>(S.a, NM0_A_SPLIT, r, 64, t);
      }
    }
    tc_fence_before();
    __syncthreads();
    {
      float d[32];
      wg_gemm6<64>(d, a_desc, [&](int sp, int kb) {
        return b_desc_ex(w_saddr + NM0_W6_BASE + sp * NM0_W6_SPLIT + kb * 2048, 1024, 128); }, 5, false);
      __syncthreads();
      wg_store_d<64>(dtile + wgi * 64 * NM0_LD, NM0_LD, d, tid & 127);
    }
    __syncthreads();
    {
      float v[32];
      tile_ld32f(dtile, NM0_LD, r, half * 32, v);
#pragma unroll
      for (int c = 0; c < 32; ++c) v[c] += cst.b6[half * 32 + c];
      if (valid) {
        float4* o = reinterpret_cast<float4*>(h_out + (long)node * EQD_HID + half * 32);
#pragma unroll
        for (int c4 = 0; c4 < 8; ++c4) o[c4] = make_float4(v[c4 * 4], v[c4 * 4 + 1], v[c4 * 4 + 2], v[c4 * 4 + 3]);
      }
    }
    __syncthreads();   // the result tile has been read: the region takes the next tile's A operand
  }
  TRACE_END(3);
}

}  // namespace eqd

EQD_TRACE_SETTER(eqd_trace_set_mlp)

extern "C" int eqd_node_mlp_tc(const eqd_graph* g, const eqd_layer* p_l, const float* h_in, const float* aggr,
                               const float* mu, const float* h0, float* h_out, void* stream) {
  const eqd_layer_params* p = p_l ? &p_l->dev : nullptr;
  if (!g || !p || !h_in || !aggr || !mu || !h0 || !h_out) return EQD_ERR_BAD_ARG;
  if (p->dh != 64 || p->dhp != 64) return EQD_ERR_UNSUPPORTED;
  if (!(p->leaky_slope >= 0.f && p->leaky_slope <= 1.f)) return EQD_ERR_UNSUPPORTED;  // lrelu() = max(v, slope*v)
  if (!p->w_node_tc || (reinterpret_cast<uintptr_t>(p->w_node_tc) & 15)) return EQD_ERR_BAD_ARG;
  if (g->n_nodes <= 0) return EQD_OK;
  eqd::NmConsts cst;
  memcpy(&cst, p_l->consts.node, sizeof(cst));
  int ntiles = (g->n_nodes + EQD_TM - 1) / EQD_TM;
  size_t smem = sizeof(eqd::NmSmem) + 128;
  EQD_SET_SMEM((eqd::node_mlp_tc_kernel), smem);
  int grid = ntiles < EQD_SMS ? ntiles : EQD_SMS;
  eqd::node_mlp_tc_kernel<<<grid, NM_THREADS, smem, (cudaStream_t)stream>>>(g->n_nodes, *p, cst, h_in, aggr, mu, h0, h_out);
  EQD_CUDA_LAUNCH_CHECK();
  return EQD_OK;
}

extern "C" int eqd_node_mlp_tc0(const eqd_graph* g, const eqd_layer* p_l, const float* h0, const float* aggr,
                                const float* mu, float* h_out, void* stream) {
  const eqd_layer_params* p = p_l ? &p_l->dev : nullptr;
  if (!g || !p || !h0 || !aggr || !mu || !h_out) return EQD_ERR_BAD_ARG;
  if (p->dh != 69 || p->dhp != 72) return EQD_ERR_UNSUPPORTED;
  if (!(p->leaky_slope >= 0.f && p->leaky_slope <= 1.f)) return EQD_ERR_UNSUPPORTED;  // lrelu() = max(v, slope*v)
  if (!p->w_node_tc || (reinterpret_cast<uintptr_t>(p->w_node_tc) & 15)) return EQD_ERR_BAD_ARG;
  if (g->n_nodes <= 0) return EQD_OK;
  eqd::Nm0Consts cst;
  memcpy(&cst, p_l->consts.node, sizeof(cst));
  int ntiles = (g->n_nodes + EQD_TM - 1) / EQD_TM;
  size_t smem = sizeof(eqd::Nm0Smem) + 128;
  EQD_SET_SMEM((eqd::node_mlp0_tc_kernel), smem);
  int grid = ntiles < EQD_SMS ? ntiles : EQD_SMS;
  eqd::node_mlp0_tc_kernel<<<grid, NM_THREADS, smem, (cudaStream_t)stream>>>(g->n_nodes, *p, cst, h0, aggr, mu, h_out);
  EQD_CUDA_LAUNCH_CHECK();
  return EQD_OK;
}

extern "C" int eqd_attention_tc0(const eqd_graph*, const float*, const void*, const float*, float*, void*);

// Layer 0 (dh == 69): attention (64 tensor-core channels + 5 fp32 ones), node MLP, next layer's projections.
extern "C" int eqd_node_stage_tc0(const eqd_graph* g, const eqd_layer* p_l, const eqd_layer* p_next_l,
                                  const float* h0, const float* proj, const float* aggr, void* kv, const float* x5,
                                  float* mu, float* h_out, float* proj_next, void* stream) {
  const eqd_layer_params* p = p_l ? &p_l->dev : nullptr;
  const eqd_layer_params* p_next = p_next_l ? &p_next_l->dev : nullptr;
  if (!g || !p || !kv || !mu || !x5) return EQD_ERR_BAD_ARG;
  if (p_next && !proj_next) return EQD_ERR_BAD_ARG;
  int rc = eqd_attention_tc0(g, proj, kv, x5, mu, stream);
  if (rc) return rc;
  rc = eqd_node_mlp_tc0(g, p_l, h0, aggr, mu, h_out, stream);
  if (rc) return rc;
  if (p_next) rc = eqd_project_tc(g, p_next_l, h_out, proj_next, kv, stream);
  return rc;
}

extern "C" int eqd_project_tc(const eqd_graph*, const eqd_layer*, const float*, float*, void*, void*);
extern "C" int eqd_attention_tc(const eqd_graph*, const float*, const void*, float*, void*);

extern "C" int eqd_node_stage_tc(const eqd_graph* g, const eqd_layer* p_l, const eqd_layer* p_next_l,
                                 const float* h_in, const float* h0, const float* proj, const float* aggr, void* kv,
                                 float* mu, float* h_out, float* proj_next, void* stream) {
  const eqd_layer_params* p = p_l ? &p_l->dev : nullptr;
  const eqd_layer_params* p_next = p_next_l ? &p_next_l->dev : nullptr;
  if (!g || !p || !kv || !mu) return EQD_ERR_BAD_ARG;
  if (p_next && !proj_next) return EQD_ERR_BAD_ARG;
  int rc = eqd_attention_tc(g, proj, kv, mu, stream);
  if (rc) return rc;
  rc = eqd_node_mlp_tc(g, p_l, h_in, aggr, mu, h0, h_out, stream);
  if (rc) return rc;
  if (p_next) rc = eqd_project_tc(g, p_next_l, h_out, proj_next, kv, stream);
  return rc;
}
