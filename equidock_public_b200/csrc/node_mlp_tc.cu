// Node MLP of a 64-wide IEGMN layer (rigid_docking_model.py:319-337) on the tensor cores (wgmma, bf16x6):
//   h' = skip( W6 . LayerNorm(LeakyReLU(W5 . [h | aggr_msg | mu | h0] + b5)) + b6 )
// Weight-stationary: W5 (64 x 272) and W6 (64 x 64) as bf16x3 panels, 126 KB in shared memory for the life of the CTA.
// node_mlp_tc_kernel (the 64-wide layers) runs warpgroup tile chains; node_mlp0_tc_kernel (layer 0) 128-row tiles.
#include "tc_common.cuh"

namespace eqd {

#define NM_THREADS 256
#define NM_W5_SPLIT 34816   // 64 x 272 bf16
#define NM_W6_BASE 104448
#define NM_W6_SPLIT 8192
#define NM_W_BYTES 129024

struct NmConsts { float b5[64], ln_g[64], ln_b[64], b6[64]; };

// ---- the 64-wide layers -------------------------------------------------------------------------------------------------
// One persistent CTA of NM_CHAINS warpgroups per SM sharing the resident panels.  Each warpgroup runs its own chain of
// 64-row tiles and synchronises only inside itself (its named barrier).  The 272-wide input of node_mlp.0 arrives in five
// K-pieces: h, aggr, mu and h0[0:64] stream through the chain's ring of NM_SLOTS staging buffers by cp.async, two pieces
// ahead of their use and across tile boundaries, and each becomes bf16x3 RS A fragments; h0[64:72] plus 8 zero channels
// (one k-block) is read from global memory straight into A fragments.  Each piece is a fresh accumulation summed into the
// accumulator fragments with round-to-nearest adds.  Bias, LeakyReLU and the LayerNorm run on the fragments (row
// statistics over the quad, in the chain order of a row-per-thread epilogue), which then feed node_mlp.4 as RS A
// fragments; the skip line takes h from the registers of piece 0 and h' leaves by direct fragment stores (a quad writes
// 32 contiguous bytes of a row).  Every element of h' takes the splits, products, order and epilogue of the 128-row kernel
// this one replaced, with the same multiply-add contraction (pinned below with the _rn intrinsics).
// P = 3 (bf16x3): two-term A splits and the three leading products in both GEMMs.
#define NM_CHAINS 2
#define NM_SLOTS 3   // staging buffers per chain: pieces are issued NM_SLOTS - 1 ahead

struct NmSmem {
  unsigned char w[NM_W_BYTES];
  float stage[NM_CHAINS][NM_SLOTS][64 * 64];   // 64 rows x 64 channels of a piece (16-byte chunks swizzled, stage_rows64)
  float c[256];                                // b5 | ln_g | ln_b | b6
  unsigned long long w_bar;
};

// Bytes of dynamic shared memory past NmSmem: the final LayerNorm's gamma | beta (HLN only)
#define NM_HLN_BYTES 512
static_assert(sizeof(NmSmem) + 128 + NM_HLN_BYTES <= 232448, "node MLP shared memory exceeds the sm_90 limit");

// HLN: the final feature LayerNorm (final_h_layernorm_layer of eqd_layer_norms `nm`) on the row after the skip combination,
// statistics over the quad as for node_mlp.3 (quad_ln_stats), the last step before h' is stored.
template <int P, bool HLN>
__global__ void __launch_bounds__(NM_CHAINS * 128, 1)
node_mlp_tc_kernel(int n_nodes, eqd_layer_params p, const __grid_constant__ NmConsts cst, const float* __restrict__ h_in,
                   const float* __restrict__ aggr, const float* __restrict__ mu, const float* __restrict__ h0,
                   float* __restrict__ h_out, eqd_layer_norms nm) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  NmSmem& S = *reinterpret_cast<NmSmem*>(smem_raw);
  float* hln = reinterpret_cast<float*>(smem_raw + sizeof(NmSmem));   // [gamma 64 | beta 64]
  const int tid = threadIdx.x, wgi = tid >> 7, t = tid & 127, lane = t & 31;
  float (&ring)[NM_SLOTS][64 * 64] = S.stage[wgi];
  const int bar = 1 + wgi;   // this chain's named barrier
  const int ntiles = (n_nodes + 63) / 64, tstride = gridDim.x * NM_CHAINS, tile0 = blockIdx.x * NM_CHAINS + wgi;
  if (tid == 0) {
    mbar_init(&S.w_bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    mbar_expect_tx(&S.w_bar, NM_W_BYTES);
    bulk_g2s(S.w, p.w_node_tc, NM_W_BYTES, &S.w_bar);
  }
  for (int i = tid; i < 256; i += NM_CHAINS * 128) S.c[i] = reinterpret_cast<const float*>(&cst)[i];
  if (HLN && tid < 128) hln[tid] = tid < 64 ? nm.final_ln_g[tid] : nm.final_ln_b[tid - 64];
  __syncthreads();
  const unsigned w_saddr = smem_u32(S.w);
  const float slope = p.leaky_slope, sk = p.skip_weight_h, sk1 = 1.f - p.skip_weight_h;
  // accumulator-fragment rows of this thread: fr0 and fr0 + 8; columns 8 j + fc + {0, 1}, j = 0..7
  const int fr0 = (t >> 5) * 16 + (lane >> 2), fc = 2 * (lane & 3);

  // piece q of the chain's stream: piece q & 3 (h, aggr, mu, h0[0:64]) of its tile number q >> 2, into slot q % NM_SLOTS;
  // one commit group per piece (empty past the last tile), so cp_async_wait<NM_SLOTS - 2> waits for piece q alone
  auto issue = [&](int q) {
    const int tile = tile0 + (q >> 2) * tstride, pc = q & 3;
    if (tile < ntiles) {
      const float* src = pc == 0 ? h_in : pc == 1 ? aggr : pc == 2 ? mu : h0;
      stage_rows64(ring[q % NM_SLOTS], src, pc == 3 ? EQD_H0_PAD : EQD_HID, 0, (long)tile * 64, min(64, n_nodes - tile * 64), t);
    } else {
      cp_async_commit();
    }
  };
  int q = 0;
  for (int i = 0; i < NM_SLOTS - 1; ++i) issue(i);
  mbar_wait(&S.w_bar, 0);

  for (int tile = tile0; tile < ntiles; tile += tstride) {
    const int node0 = tile * 64, nvalid = min(64, n_nodes - node0);
    // piece 4 (h0[64:72]): A registers 0, 1 of the k-block = channels 64 + fc + {0, 1} of rows fr0, fr0 + 8
    float2 x4[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int row = fr0 + 8 * hh;
      x4[hh] = row < nvalid ? *reinterpret_cast<const float2*>(h0 + (long)(node0 + row) * EQD_H0_PAD + 64 + fc)
                            : make_float2(0.f, 0.f);
    }
    // ---- node_mlp.0 over [h | aggr | mu | h0] in 5 K-pieces ---------------------------------------------------------
    float acc[32], hs[32];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float2 bj = *reinterpret_cast<const float2*>(&S.c[8 * j + fc]);
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        acc[4 * j + 2 * hh] = bj.x;
        acc[4 * j + 2 * hh + 1] = bj.y;
      }
    }
#pragma unroll 1   // unrolled, ptxas serialises the wgmmas (C7511: too few registers for the pipeline)
    for (int pc = 0; pc < 4; ++pc, ++q) {
      cp_async_wait<NM_SLOTS - 2>();
      wg_barrier(bar);   // piece q has landed, and every thread is done with piece q - 1's slot
      issue(q + NM_SLOTS - 1);
      float v[32];
      staged_rows_to_frag(ring[q % NM_SLOTS], t, v);
      if (pc == 0) {
#pragma unroll
        for (int i = 0; i < 32; ++i) hs[i] = v[i];   // the skip operand
      }
      unsigned af[3][4][4];
      acc_to_a_split3<4, P>(v, af);
      float d[32];
      wg_gemm6_rs_issue<64, 4, 0, false, P>(d, af, [&](int sp, int kb) {
        return b_desc_ex(w_saddr + (4 * pc + kb) * 2048 + sp * NM_W5_SPLIT, 1024, 128); }, false);
      wg_mma_wait(d);
#pragma unroll
      for (int i = 0; i < 32; ++i) acc[i] = __fadd_rn(acc[i], d[i]);
    }
    {
      unsigned a4[3][1][4];
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) split3_pair<P>(x4[hh].x, x4[hh].y, a4[0][0][hh], a4[1][0][hh], a4[2][0][hh]);
#pragma unroll
      for (int sp = 0; sp < 3; ++sp) a4[sp][0][2] = a4[sp][0][3] = 0u;
      float d[32];
      wg_gemm6_rs_issue<64, 1, 0, false, P>(d, a4, [&](int sp, int kb) {
        return b_desc_ex(w_saddr + 16 * 2048 + sp * NM_W5_SPLIT, 1024, 128); }, false);
      wg_mma_wait(d);
#pragma unroll
      for (int i = 0; i < 32; ++i) acc[i] = __fadd_rn(acc[i], d[i]);
    }
    // ---- LeakyReLU, LayerNorm -> bf16x3 A fragments ; node_mlp.4 ----------------------------------------------------
    unsigned af[3][4][4];
    {
      float (&v)[32] = acc;
#pragma unroll
      for (int i = 0; i < 32; ++i) v[i] = fmaxf(v[i], __fmul_rn(v[i], slope));
      // per 32-column half ch, two-pass (mean_ch, M2_ch) over four chains, then the Chan et al. combination
      // mean = (m0 + m1) / 2, M2 = M2_0 + M2_1 + (m0 - m1)^2 * 16
      float pv[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) pv[i] = __shfl_xor_sync(0xffffffffu, v[i], 2);
      float msum[2], rstd[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float mh[2], qh[2];
#pragma unroll
        for (int ch = 0; ch < 2; ++ch) {
          float s0 = 0.f, s1 = 0.f;
#pragma unroll
          for (int c4 = 0; c4 < 8; ++c4) {
            s0 = __fadd_rn(s0, chain_val(v, pv, h, ch, c4, 0));
            s1 = __fadd_rn(s1, chain_val(v, pv, h, ch, c4, 1));
          }
          const float sp = __fadd_rn(s0, s1);
          mh[ch] = __fmul_rn(__fadd_rn(sp, __shfl_xor_sync(0xffffffffu, sp, 1)), 1.f / 32.f);
          float q0 = 0.f, q1 = 0.f;
#pragma unroll
          for (int c4 = 0; c4 < 8; ++c4) {
            const float d0 = __fadd_rn(chain_val(v, pv, h, ch, c4, 0), -mh[ch]);
            const float d1 = __fadd_rn(chain_val(v, pv, h, ch, c4, 1), -mh[ch]);
            q0 = __fmaf_rn(d0, d0, q0);
            q1 = __fmaf_rn(d1, d1, q1);
          }
          const float qp = __fadd_rn(q0, q1);
          qh[ch] = __fadd_rn(qp, __shfl_xor_sync(0xffffffffu, qp, 1));
        }
        msum[h] = __fadd_rn(mh[0], mh[1]);
        const float dm = __fadd_rn(mh[0], -mh[1]);
        const float var = __fmaf_rn(__fmul_rn(dm, dm), 16.f, __fadd_rn(qh[0], qh[1]));
        rstd[h] = 1.f / sqrtf(__fmaf_rn(var, 1.f / 64.f, 1e-5f));
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float2 gj = *reinterpret_cast<const float2*>(&S.c[64 + 8 * j + fc]);
        const float2 bj = *reinterpret_cast<const float2*>(&S.c[128 + 8 * j + fc]);
#pragma unroll
        for (int h = 0; h < 2; ++h) {   // v - mean as v - 0.5 (m0 + m1) in one rounding
          float& x0 = v[4 * j + 2 * h];
          float& x1 = v[4 * j + 2 * h + 1];
          x0 = __fmaf_rn(__fmul_rn(__fmaf_rn(msum[h], -0.5f, x0), rstd[h]), gj.x, bj.x);
          x1 = __fmaf_rn(__fmul_rn(__fmaf_rn(msum[h], -0.5f, x1), rstd[h]), gj.y, bj.y);
        }
      }
      acc_to_a_split3<4, P>(v, af);
    }
    {
      float d[32];
      wg_gemm6_rs_issue<64, 4, 0, false, P>(d, af, [&](int sp, int kb) {
        return b_desc_ex(w_saddr + NM_W6_BASE + sp * NM_W6_SPLIT + kb * 2048, 1024, 128); }, false);
      wg_mma_wait(d);
      if (HLN) {   // y = skip(...) for every fragment row (the quad reductions need all of them), then LN_f, store
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float2 bj = *reinterpret_cast<const float2*>(&S.c[192 + 8 * j + fc]);
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            const int i = 4 * j + 2 * hh;
            d[i] = __fmaf_rn(__fadd_rn(d[i], bj.x), sk, __fmul_rn(hs[i], sk1));
            d[i + 1] = __fmaf_rn(__fadd_rn(d[i + 1], bj.y), sk, __fmul_rn(hs[i + 1], sk1));
          }
        }
        float mean[2], rstd[2];
        quad_ln_stats(d, mean, rstd);
        quad_ln_apply(d, mean, rstd, hln, hln + 64, fc);
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int row = fr0 + 8 * hh;
          if (row < nvalid) {
            float* o = h_out + (long)(node0 + row) * EQD_HID + fc;
#pragma unroll
            for (int j = 0; j < 8; ++j)
              *reinterpret_cast<float2*>(o + 8 * j) = make_float2(d[4 * j + 2 * hh], d[4 * j + 2 * hh + 1]);
          }
        }
      } else
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int row = fr0 + 8 * hh;
        if (row < nvalid) {
          float* o = h_out + (long)(node0 + row) * EQD_HID + fc;
#pragma unroll
          for (int j = 0; j < 8; ++j) {   // :332-334
            const float2 bj = *reinterpret_cast<const float2*>(&S.c[192 + 8 * j + fc]);
            const int i = 4 * j + 2 * hh;
            *reinterpret_cast<float2*>(o + 8 * j) =
                make_float2(__fmaf_rn(__fadd_rn(d[i], bj.x), sk, __fmul_rn(hs[i], sk1)),
                            __fmaf_rn(__fadd_rn(d[i + 1], bj.y), sk, __fmul_rn(hs[i + 1], sk1)));
          }
        }
      }
    }
  }
  cp_async_wait<0>();
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

// HLN: the final feature LayerNorm (eqd_layer_norms `nm`) on node_mlp's output (layer 0 has no skip), its row statistics
// over the two halves of a row through `red`, the last step before h' is stored.
template <bool HLN>
__global__ void __launch_bounds__(NM_THREADS, 1)
node_mlp0_tc_kernel(int n_nodes, eqd_layer_params p, const __grid_constant__ Nm0Consts cst, const float* __restrict__ h0,
                    const float* __restrict__ aggr, const float* __restrict__ mu /*[n][72]*/, float* __restrict__ h_out,
                    eqd_layer_norms nm) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  Nm0Smem& S = *reinterpret_cast<Nm0Smem*>(smem_raw);
  const int tid = threadIdx.x, q = tid, half = q >> 7, r = q & 127, wgi = tid >> 7;
  const int ntiles = (n_nodes + EQD_TM - 1) / EQD_TM;
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
      if (HLN) {   // final_h_layernorm_layer: two-pass row statistics of the 64 outputs, half rows combined in red
        float s = 0.f;
#pragma unroll
        for (int c = 0; c < 32; ++c) s += v[c];
        red[(r * 2 + half) * 2] = s;
        __syncthreads();
        const float mean = (red[r * 4] + red[r * 4 + 2]) * (1.f / 64.f);
        float q = 0.f;
#pragma unroll
        for (int c = 0; c < 32; ++c) {
          const float dv = v[c] - mean;
          q = fmaf(dv, dv, q);
        }
        red[(r * 2 + half) * 2 + 1] = q;
        __syncthreads();
        const float rstd = 1.f / sqrtf((red[r * 4 + 1] + red[r * 4 + 3]) * (1.f / 64.f) + 1e-5f);
#pragma unroll
        for (int c = 0; c < 32; ++c) v[c] = (v[c] - mean) * rstd * nm.final_ln_g[half * 32 + c] + nm.final_ln_b[half * 32 + c];
      }
      if (valid) {
        float4* o = reinterpret_cast<float4*>(h_out + (long)node * EQD_HID + half * 32);
#pragma unroll
        for (int c4 = 0; c4 < 8; ++c4) o[c4] = make_float4(v[c4 * 4], v[c4 * 4 + 1], v[c4 * 4 + 2], v[c4 * 4 + 3]);
      }
    }
    __syncthreads();   // the result tile has been read: the region takes the next tile's A operand
  }
}

template <int P, bool HLN>
static int launch_node_mlp_tc(const eqd_graph* g, const eqd_layer* p_l, const float* h_in, const float* aggr,
                              const float* mu, const float* h0, float* h_out, void* stream) {
  NmConsts cst;
  memcpy(&cst, p_l->consts.node, sizeof(cst));
  const int ntiles = (g->n_nodes + 63) / 64;
  const size_t smem = sizeof(NmSmem) + 128 + (HLN ? NM_HLN_BYTES : 0);
  EQD_SET_SMEM((node_mlp_tc_kernel<P, HLN>), smem);
  int grid = (ntiles + NM_CHAINS - 1) / NM_CHAINS;
  if (grid > EQD_SMS) grid = EQD_SMS;
  node_mlp_tc_kernel<P, HLN><<<grid, NM_CHAINS * 128, smem, (cudaStream_t)stream>>>(g->n_nodes, p_l->dev, cst, h_in, aggr,
                                                                                   mu, h0, h_out, p_l->norms);
  EQD_CUDA_LAUNCH_CHECK();
  return EQD_OK;
}

}  // namespace eqd

extern "C" int eqd_node_mlp_tc(const eqd_graph* g, const eqd_layer* p_l, const float* h_in, const float* aggr,
                               const float* mu, const float* h0, float* h_out, void* stream) {
  const eqd_layer_params* p = p_l ? &p_l->dev : nullptr;
  if (!g || !p || !h_in || !aggr || !mu || !h0 || !h_out) return EQD_ERR_BAD_ARG;
  if (p_l->dropout.p > 0.f) return EQD_ERR_UNSUPPORTED;   // dropout runs on the fp32 node stage (eqd_node_stage)
  if (p->dh != 64 || p->dhp != 64) return EQD_ERR_UNSUPPORTED;
  if (!(p->leaky_slope >= 0.f && p->leaky_slope <= 1.f)) return EQD_ERR_UNSUPPORTED;  // lrelu() = max(v, slope*v)
  const int products = eqd_mma_products(p);
  if (!products) return EQD_ERR_UNSUPPORTED;
  if (!p->w_node_tc || (reinterpret_cast<uintptr_t>(p->w_node_tc) & 15)) return EQD_ERR_BAD_ARG;
  const int hln = eqd_final_ln(p_l);
  if (hln < 0) return EQD_ERR_BAD_ARG;
  if (g->n_nodes <= 0) return EQD_OK;
  if (hln)
    return products == 3 ? eqd::launch_node_mlp_tc<3, true>(g, p_l, h_in, aggr, mu, h0, h_out, stream)
                         : eqd::launch_node_mlp_tc<6, true>(g, p_l, h_in, aggr, mu, h0, h_out, stream);
  return products == 3 ? eqd::launch_node_mlp_tc<3, false>(g, p_l, h_in, aggr, mu, h0, h_out, stream)
                       : eqd::launch_node_mlp_tc<6, false>(g, p_l, h_in, aggr, mu, h0, h_out, stream);
}

extern "C" int eqd_node_mlp_tc0(const eqd_graph* g, const eqd_layer* p_l, const float* h0, const float* aggr,
                                const float* mu, float* h_out, void* stream) {
  const eqd_layer_params* p = p_l ? &p_l->dev : nullptr;
  if (!g || !p || !h0 || !aggr || !mu || !h_out) return EQD_ERR_BAD_ARG;
  if (p_l->dropout.p > 0.f) return EQD_ERR_UNSUPPORTED;   // dropout runs on the fp32 node stage (eqd_node_stage)
  if (p->dh != 69 || p->dhp != 72 || !eqd_mma_products(p)) return EQD_ERR_UNSUPPORTED;
  if (!(p->leaky_slope >= 0.f && p->leaky_slope <= 1.f)) return EQD_ERR_UNSUPPORTED;  // lrelu() = max(v, slope*v)
  if (!p->w_node_tc || (reinterpret_cast<uintptr_t>(p->w_node_tc) & 15)) return EQD_ERR_BAD_ARG;
  const int hln = eqd_final_ln(p_l);
  if (hln < 0) return EQD_ERR_BAD_ARG;
  if (g->n_nodes <= 0) return EQD_OK;
  eqd::Nm0Consts cst;
  memcpy(&cst, p_l->consts.node, sizeof(cst));
  int ntiles = (g->n_nodes + EQD_TM - 1) / EQD_TM;
  size_t smem = sizeof(eqd::Nm0Smem) + 128;
  int grid = ntiles < EQD_SMS ? ntiles : EQD_SMS;
  if (hln) {
    EQD_SET_SMEM((eqd::node_mlp0_tc_kernel<true>), smem);
    eqd::node_mlp0_tc_kernel<true><<<grid, NM_THREADS, smem, (cudaStream_t)stream>>>(g->n_nodes, *p, cst, h0, aggr, mu, h_out,
                                                                                    p_l->norms);
  } else {
    EQD_SET_SMEM((eqd::node_mlp0_tc_kernel<false>), smem);
    eqd::node_mlp0_tc_kernel<false><<<grid, NM_THREADS, smem, (cudaStream_t)stream>>>(g->n_nodes, *p, cst, h0, aggr, mu,
                                                                                     h_out, p_l->norms);
  }
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
  if (!eqd_mma_products(p)) return EQD_ERR_UNSUPPORTED;   // layer 0 runs bf16x6 only
  int rc = eqd_attention_tc0(g, proj, kv, x5, mu, stream);
  if (rc) return rc;
  rc = eqd_node_mlp_tc0(g, p_l, h0, aggr, mu, h_out, stream);
  if (rc) return rc;
  if (p_next) rc = eqd_project_tc(g, p_next_l, h_out, proj_next, kv, stream);
  return rc;
}

extern "C" int eqd_project_tc(const eqd_graph*, const eqd_layer*, const float*, float*, void*, void*);
int eqd_attention_tc_products(const eqd_graph*, const float*, const void*, float*, int, void*);

// Attention and node MLP take this layer's product count, the next layer's projections that of p_next.

extern "C" int eqd_node_stage_tc(const eqd_graph* g, const eqd_layer* p_l, const eqd_layer* p_next_l,
                                 const float* h_in, const float* h0, const float* proj, const float* aggr, void* kv,
                                 float* mu, float* h_out, float* proj_next, void* stream) {
  const eqd_layer_params* p = p_l ? &p_l->dev : nullptr;
  const eqd_layer_params* p_next = p_next_l ? &p_next_l->dev : nullptr;
  if (!g || !p || !kv || !mu) return EQD_ERR_BAD_ARG;
  if (p_next && !proj_next) return EQD_ERR_BAD_ARG;
  const int products = eqd_mma_products(p);
  if (!products) return EQD_ERR_UNSUPPORTED;
  int rc = eqd_attention_tc_products(g, proj, kv, mu, products, stream);
  if (rc) return rc;
  rc = eqd_node_mlp_tc(g, p_l, h_in, aggr, mu, h0, h_out, stream);
  if (rc) return rc;
  if (p_next) rc = eqd_project_tc(g, p_next_l, h_out, proj_next, kv, stream);
  return rc;
}
