// Edge stage of IEGMN_Layer.forward (rigid_docking_model.py:204-237, 263-292) on the tensor cores (wgmma),
// fp32-accurate through a 3-way bf16 split of both operands ("bf16x6": a*w ~ a0w0 + a0w1 + a1w0 + a0w2 + a1w1 + a2w0,
// fp32 accumulation).
//
// One persistent CTA of three warpgroups per SM.  Each warpgroup owns its own tiles of <= 64 edges (tn destination nodes)
// and runs them as an independent chain that synchronises only inside the warpgroup (named barriers, its own mbarrier),
// so some warpgroups' epilogues run while another's MMAs occupy the tensor pipe.  The weight panels are shared.  Per tile:
//   indices, row_ptr, x[src], x[dst] (cp.async) and he rows (cp.async.bulk) were prefetched during the previous tile
//   he rows + 15 RBFs -> [he|rbf] bf16x3 -> smem (2 threads per row)          A operand of GEMM1 (K=48)
//   Psrc[src], Pdst[dst] -> registers in the accumulator layout (read from L2 under the A build and GEMM1)
//   GEMM1 (18 wgmma, A and B = edge_mlp.0.weight[:, 2dh:] bf16x3 in smem; the next tile's prefetch is issued under it)
//     -> epilogue 1 on the accumulator fragments: (acc + Psrc) + Pdst, LeakyReLU, LayerNorm (a row's 64 columns sit on
//        the 4 lanes of a quad: lane shuffles) -> bf16x3 A fragments in registers
//   GEMM2 and GEMM3 as RS wgmma on those fragments (2 x 24, N=64 halves of the stacked panel [W2 ; W3 W2])
//     -> msg (+b2) -> fp32 tile in smem (mean aggregation at the destination nodes)
//     -> coordinate MLP hidden layer -> LeakyReLU, (coordinate LayerNorm,) dot w4 -> phi (lane shuffles);
//        x' = eta x0 + (1-eta) x + mean(x_rel phi) in fp64.
// Per-edge activations never leave the SM; weights are read from HBM/L2 once per CTA.  A tile whose nodes all have 10
// in-edges (a k-NN graph) needs no row_ptr lookups in the aggregation.
//
// Rounding: every step is that of a row-per-thread epilogue on shared-memory operands: the split, the six products, their
// order and the accumulation chain of every GEMM output, the Psrc/Pdst add order, the LayerNorm and phi summation chains
// (chain_val), the two-chain mean aggregation and the fp64 coordinate update.
// P = 3 (bf16x3, eqd_layer_params.mma_products): the same kernel with two-term A splits and the three leading products.
#include "tc_common.cuh"

namespace eqd {
#define TC_WGS 3              // warpgroups per CTA, one tile chain each
#define TC_THREADS (128 * TC_WGS)
#define TC_ROWS 64            // edge rows per warpgroup tile
#define TC_MAX_TN 32          // destination nodes per tile
#define TC_LD 72              // fp32 row stride of the msg tile (72 % 32 = 8: the fragment stores are conflict-free)
#define TC_W_BYTES 67584      // 3 splits x (6144 + 8192 + 8192)
#define TC_W1_SPLIT 6144
#define TC_W23_BASE 18432    // [W2 ; W3 W2] stacked, N = 128
#define TC_W23_SPLIT 16384
#define TC_HE_FLOATS (TC_ROWS * EQD_EDGE_FEATS + 16)
#define TC_A_SPLIT 6144       // A operand of GEMM1: 64 rows x K = 48 bf16 per split

struct __align__(128) TcWgSmem {          // one warpgroup's tile chain
  unsigned char a[3 * TC_A_SPLIT];        // [he|rbf] A operand (bf16x3), canonical no-swizzle layout
  float msg[TC_ROWS * TC_LD];             // msg + b2 per edge row
  float he[TC_HE_FLOATS];                 // raw he rows of the tile (bulk-copied, 16B-aligned chunks)
  double xs[2][TC_ROWS * 6];              // x[src], x[dst] of the tile's edges (prefetched one tile ahead)
  double xm[TC_ROWS * 3];                 // x_rel per edge
  double phi[TC_ROWS];                    // phi + b_coor2 per edge
  int src[2][TC_ROWS];
  int dst[2][TC_ROWS];
  int rp[2][TC_MAX_TN + 4];
  unsigned long long he_bar;
};

struct EdgeConsts {                       // per-layer vectors, passed by value and staged in smem
  float ln_g[64], ln_b[64], b2[64], b3[64], w4[64];
};

struct TcSmem {
  unsigned char w[TC_W_BYTES];            // bf16x3 weights, canonical K-major no-swizzle layout
  TcWgSmem wg[TC_WGS];
  EdgeConsts cst;
  unsigned long long w_bar;
};

// Bytes of dynamic shared memory past TcSmem: the coordinate LayerNorm's gamma | beta (CLN only)
#define TC_CLN_BYTES 512
static_assert(sizeof(TcSmem) + 128 + TC_CLN_BYTES <= 232448, "edge stage shared memory exceeds the sm_90 limit");

// CLN: the coordinate LayerNorm coors_mlp.3 (eqd_layer_norms `nm`) on LeakyReLU(hidden + b3), with the statistics and
// order of edge_mlp.3, before the dot product with w4.
template <int P, bool CLN>
__global__ void __launch_bounds__(TC_THREADS, 1)
edge_stage_tc_kernel(eqd_graph g, eqd_layer_params p, const __grid_constant__ EdgeConsts cst_p,
                     const float* __restrict__ proj, const double* __restrict__ x_in, const double* __restrict__ x_orig,
                     float* __restrict__ aggr, double* __restrict__ x_out, int* __restrict__ status, int tn,
                     eqd_layer_norms nm) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  TcSmem& S = *reinterpret_cast<TcSmem*>(smem_raw);
  float* cln = reinterpret_cast<float*>(smem_raw + sizeof(TcSmem));   // [gamma 64 | beta 64]
  const int tid = threadIdx.x, wgi = tid >> 7, t = tid & 127, r = t & 63, half = t >> 6;
  const int warp = t >> 5, lane = t & 31;
  TcWgSmem& W = S.wg[wgi];
  const EdgeConsts& cst = S.cst;
  const int bar = 1 + wgi;               // this warpgroup's named barrier
  const int pw = 128 + 3 * p.dhp;
  const int ntiles = (g.n_nodes + tn - 1) / tn;
  const float slope = p.leaky_slope;

  // ---- one-time setup: barriers, weights (one TMA bulk copy), per-layer vectors ------------------------------------
  if (tid == 0) {
    mbar_init(&S.w_bar, 1);
    for (int w = 0; w < TC_WGS; ++w) mbar_init(&S.wg[w].he_bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    mbar_expect_tx(&S.w_bar, TC_W_BYTES);
    bulk_g2s(S.w, p.w_edge_tc, TC_W_BYTES, &S.w_bar);
  }
  for (int i = tid; i < 5 * 64; i += TC_THREADS) (&S.cst.ln_g[0])[i] = (&cst_p.ln_g[0])[i];
  if (CLN && tid < 128) cln[tid] = tid < 64 ? nm.coors_ln_g[tid] : nm.coors_ln_b[tid - 64];
  __syncthreads();
  mbar_wait(&S.w_bar, 0);
  unsigned he_phase = 0;
  const unsigned w_saddr = smem_u32(S.w), a_saddr = smem_u32(W.a);
  auto a_desc = [&](int sp, int kb) { return a_desc_at<TC_ROWS>(a_saddr, TC_A_SPLIT, 0, sp, kb); };

  // Prefetch of a tile's indices, row_ptr and he rows (e0 = row_ptr[n0], e1 = row_ptr[n0 + nn] read ahead by the caller).
  auto prefetch = [&](int tile, int buf, int e0, int e1, int& off_l, int& n_l, int& off_r) {
    const int n0 = tile * tn, nn = min(tn, g.n_nodes - n0);
    const int ne = e1 - e0;
    off_l = off_r = 0;
    n_l = 0;
    if (ne <= TC_ROWS) {
      if (r < ne) {   // every thread fetches the index its own prefetch_x() reads (no barrier in between)
        if (half == 0) cp_async4(&W.src[buf][r], g.col_src + e0 + r);
        else cp_async4(&W.dst[buf][r], g.edge_dst + e0 + r);
      }
      if (half == 0 && r <= nn) cp_async4(&W.rp[buf][r], g.row_ptr + n0 + r);
      // he rows: [e0, e1) split at the ligand/receptor array boundary; 16-byte aligned bulk copies
      const int el0 = min(e0, g.n_lig_edges), el1 = min(e1, g.n_lig_edges);
      n_l = el1 - el0;
      long sl = 0, sr = 0;
      unsigned bl = 0, br = 0;
      if (n_l > 0) {
        long b0 = (long)el0 * (EQD_EDGE_FEATS * 4), b1 = (long)el1 * (EQD_EDGE_FEATS * 4);
        sl = b0 & ~15L;
        bl = (unsigned)(((b1 + 15) & ~15L) - sl);
        off_l = (int)((b0 - sl) >> 2);
      }
      const int nr = ne - n_l;
      const unsigned dst_r_off = bl;  // receptor part lands after the ligand part (bl is a multiple of 16)
      if (nr > 0) {
        long b0 = (long)(e0 + n_l - g.n_lig_edges) * (EQD_EDGE_FEATS * 4), b1 = (long)(e1 - g.n_lig_edges) * (EQD_EDGE_FEATS * 4);
        sr = b0 & ~15L;
        br = (unsigned)(((b1 + 15) & ~15L) - sr);
        off_r = (int)(dst_r_off >> 2) + (int)((b0 - sr) >> 2);
      }
      if (t == 0) {
        mbar_expect_tx(&W.he_bar, bl + br);
        if (bl) bulk_g2s(W.he, reinterpret_cast<const unsigned char*>(g.he_lig) + sl, bl, &W.he_bar);
        if (br) bulk_g2s(reinterpret_cast<unsigned char*>(W.he) + dst_r_off, reinterpret_cast<const unsigned char*>(g.he_rec) + sr, br,
                         &W.he_bar);
      }
    }
    cp_async_commit();
  };
  // Coordinates of a tile's edge endpoints -> smem (needs that tile's indices to have landed).
  auto prefetch_x = [&](int b, int ne_t) {
    if (r < ne_t && ne_t <= TC_ROWS) {
      const double* xp = x_in + (long)(half == 0 ? W.src[b][r] : W.dst[b][r]) * 3;
#pragma unroll
      for (int c = 0; c < 3; ++c) cp_async8(&W.xs[b][r * 6 + half * 3 + c], xp + c);
    }
    cp_async_commit();
  };
  auto row_range = [&](int tile, int& e0, int& e1) {
    const int n0 = tile * tn;
    e0 = __ldg(g.row_ptr + n0);
    e1 = __ldg(g.row_ptr + n0 + min(tn, g.n_nodes - n0));
  };

  int tile = blockIdx.x * TC_WGS + wgi;
  const int tstride = gridDim.x * TC_WGS;
  int buf = 0;
  int e0 = 0, ne = 0, off_l = 0, n_l = 0, off_r = 0;
  if (tile < ntiles) {
    int e1;
    row_range(tile, e0, e1);
    ne = e1 - e0;
    prefetch(tile, buf, e0, e1, off_l, n_l, off_r);
    cp_async_wait<0>();
    prefetch_x(buf, ne);
  }
  // accumulator-fragment rows of this thread: fr0 and fr0 + 8; columns 8 j + fc + {0, 1}, j = 0..7
  const int fr0 = warp * 16 + (lane >> 2), fc = 2 * (lane & 3);

  for (; tile < ntiles; tile += tstride) {
    const int n0 = tile * tn, nn = min(tn, g.n_nodes - n0);
    const bool has_next = tile + tstride < ntiles;
    int e0n = 0, e1n = 0, off_ln = 0, n_ln = 0, off_rn = 0;
    if (has_next) row_range(tile + tstride, e0n, e1n);   // consumed behind this tile's A operand
    const int nen = e1n - e0n;
    if (ne > TC_ROWS) {  // in-degree bound violated: flag, skip (uniform per warpgroup)
      if (t == 0) atomicOr(status + g.n_pairs, EQD_STATUS_DEGREE_OVERFLOW);
      cp_async_wait<0>();
      wg_barrier(bar);
      if (has_next) {
        prefetch(tile + tstride, buf ^ 1, e0n, e1n, off_ln, n_ln, off_rn);
        cp_async_wait<0>();
        prefetch_x(buf ^ 1, nen);
      }
      e0 = e0n; ne = nen; off_l = off_ln; n_l = n_ln; off_r = off_rn; buf ^= 1;
      continue;
    }
    // The coordinate update's x_orig / x_in loads go out now and are consumed at the end of the tile.
    const int o_upd = 127 - t;                 // nn * 3 <= 96 outputs on the last threads
    const int nd_upd = o_upd / 3, comp_upd = o_upd - nd_upd * 3;
    const long gi_upd = (long)(n0 + nd_upd) * 3 + comp_upd;
    double xo_upd = 0.0, xi_upd = 0.0;
    if (o_upd < nn * 3) {
      xo_upd = x_orig[gi_upd];
      xi_upd = x_in[gi_upd];
    }
    // This tile's indices, row_ptr and coordinates have landed; the previous tile is done with xm, phi and msg.
    cp_async_wait<0>();
    wg_barrier(bar);
    // Psrc[src] / Pdst[dst] of my fragment rows -> registers; they land under the A operand build and GEMM1
    float2 ps[16], pd[16];   // [2 j + h]: row fr0 + 8 h, columns 8 j + fc + {0, 1}
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int fr = fr0 + 8 * h;
      const bool ok = fr < ne;
      const float* sp = proj + (long)(ok ? W.src[buf][fr] : 0) * pw + fc;
      const float* dp = proj + (long)(ok ? W.dst[buf][fr] : n0) * pw + 64 + fc;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        ps[2 * j + h] = __ldg(reinterpret_cast<const float2*>(sp + 8 * j));
        pd[2 * j + h] = __ldg(reinterpret_cast<const float2*>(dp + 8 * j));
      }
    }
    // ---- [he|rbf] -> A (thread (r, half): half 0 he[0..23]; half 1 he[24..26], 15 RBFs, 6 zeros) ----------------------
    const bool valid = r < ne;
    {
      float a1v[24];
      mbar_wait(&W.he_bar, he_phase);
      he_phase ^= 1;
      const float* hrow = W.he + (r < n_l ? off_l + r * EQD_EDGE_FEATS : off_r + (r - n_l) * EQD_EDGE_FEATS);
      if (half == 0) {
#pragma unroll
        for (int k = 0; k < 24; ++k) a1v[k] = valid ? hrow[k] : 0.f;
      } else {
        double rx = 0.0, ry = 0.0, rz = 0.0;
        if (valid) {  // u_sub_v :204-205
          const double* xs = W.xs[buf] + r * 6;
          rx = xs[0] - xs[3];
          ry = xs[1] - xs[4];
          rz = xs[2] - xs[5];
          W.xm[r * 3 + 0] = rx;
          W.xm[r * 3 + 1] = ry;
          W.xm[r * 3 + 2] = rz;
        }
#pragma unroll
        for (int k = 0; k < 3; ++k) a1v[k] = valid ? hrow[24 + k] : 0.f;
        const float nd2 = valid ? -(float)(rx * rx + ry * ry + rz * rz) : -INFINITY;  // :208-209; padding rows: exp2(-inf) = 0
        // exp(-d^2 / 1.5^q) :210 as ex2.approx(-d^2 * log2(e)/1.5^q): 2 instructions per RBF instead of ~20; the
        // features are <= 1 and the absolute error (<= 2e-7: 2^-22 of ex2 + the rounded scale factor) is below the
        // bf16x3 operand resolution of the GEMM they feed
        constexpr double kS[EQD_N_RBF] = {1.0, 1.5, 2.25, 3.375, 5.0625, 7.59375, 11.390625, 17.0859375, 25.62890625,
                                          38.443359375, 57.6650390625, 86.49755859375, 129.746337890625,
                                          194.6195068359375, 291.92926025390625};
#pragma unroll
        for (int j = 0; j < EQD_N_RBF; ++j)
          a1v[3 + j] = exp2f(nd2 * (float)(1.4426950408889634 / kS[j]));
#pragma unroll
        for (int k = 18; k < 24; ++k) a1v[k] = 0.f;
      }
      unsigned p0[12], p1[12], p2[12];
#pragma unroll
      for (int c = 0; c < 12; ++c) split3_pair<P>(a1v[2 * c], a1v[2 * c + 1], p0[c], p1[c], p2[c]);
#pragma unroll
      for (int j = 0; j < 3; ++j) a_store8<TC_ROWS, P>(W.a, TC_A_SPLIT, r, half * 24 + 8 * j, p0 + 4 * j, p1 + 4 * j, p2 + 4 * j);
    }
    tc_fence_before();
    // The A operand is complete and the he staging consumed.  The barrier also tells whether every node of the tile has
    // exactly 10 in-edges (the k-NN graphs of protein_utils.py:339-346): the aggregation then runs without row_ptr lookups.
    const bool deg10 = wg_barrier_and(bar, t >= nn || W.rp[buf][t + 1] - W.rp[buf][t] == 10);
    // ---- GEMM1: [he|rbf] (K=48) x W1e; epilogue 1 in registers: + Psrc + Pdst, LeakyReLU, LayerNorm -> A fragments --
    unsigned af[3][4][4];
    {
      float v[32];
      wg_gemm6_issue<64, 0, P>(v, a_desc, [&](int sp, int kb) { return b_desc_ex(w_saddr + sp * TC_W1_SPLIT + kb * 2048, 1024, 128); },
                         3, false);
      if (has_next) prefetch(tile + tstride, buf ^ 1, e0n, e1n, off_ln, n_ln, off_rn);
      wg_mma_wait(v);
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          float& x0 = v[4 * j + 2 * h];
          float& x1 = v[4 * j + 2 * h + 1];
          x0 = __fadd_rn(__fadd_rn(x0, ps[2 * j + h].x), pd[2 * j + h].x);
          x1 = __fadd_rn(__fadd_rn(x1, ps[2 * j + h].y), pd[2 * j + h].y);
          x0 = fmaxf(x0, __fmul_rn(x0, slope));
          x1 = fmaxf(x1, __fmul_rn(x1, slope));
        }
      // LayerNorm statistics in the chain order of the row-per-thread formulation: per 32-column half, two-pass
      // (mean_h, M2_h) over four chains, then mean = (m0+m1)/2, M2 = M2_0 + M2_1 + (m0-m1)^2 * 16 (Chan et al.)
      float pv[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) pv[i] = __shfl_xor_sync(0xffffffffu, v[i], 2);
      float mean[2], rstd[2];
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
          const float sp = s0 + s1;
          mh[ch] = (sp + __shfl_xor_sync(0xffffffffu, sp, 1)) * (1.f / 32.f);
          float q0 = 0.f, q1 = 0.f;
#pragma unroll
          for (int c4 = 0; c4 < 8; ++c4) {
            const float d0 = __fadd_rn(chain_val(v, pv, h, ch, c4, 0), -mh[ch]);
            const float d1 = __fadd_rn(chain_val(v, pv, h, ch, c4, 1), -mh[ch]);
            q0 = fmaf(d0, d0, q0);
            q1 = fmaf(d1, d1, q1);
          }
          const float qp = q0 + q1;
          qh[ch] = qp + __shfl_xor_sync(0xffffffffu, qp, 1);
        }
        const float m0 = mh[0], m1 = mh[1];
        mean[h] = 0.5f * (m0 + m1);
        const float dm = m0 - m1;
        const float var = (qh[0] + qh[1] + dm * dm * 16.f) * (1.f / 64.f);
        rstd[h] = 1.f / sqrtf(var + 1e-5f);
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float2 gj = *reinterpret_cast<const float2*>(&cst.ln_g[8 * j + fc]);
        const float2 bj = *reinterpret_cast<const float2*>(&cst.ln_b[8 * j + fc]);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float& x0 = v[4 * j + 2 * h];
          float& x1 = v[4 * j + 2 * h + 1];
          x0 = fmaf(__fmul_rn(__fadd_rn(x0, -mean[h]), rstd[h]), gj.x, bj.x);
          x1 = fmaf(__fmul_rn(__fadd_rn(x1, -mean[h]), rstd[h]), gj.y, bj.y);
        }
      }
      acc_to_a_split3<4, P>(v, af);
    }
    if (has_next) {
      // The next tile's x[src] / x[dst] gathers go out two GEMMs before they are needed: my own index of the next tile
      // (fetched behind GEMM1) has landed once my copy groups drain
      cp_async_wait<0>();
      prefetch_x(buf ^ 1, nen);
    }
    // ---- GEMM2 and GEMM3 from the register A fragments ------------------------------------------------------------
    // msg = W2 a1 + b2 (edge_mlp.4) and the coordinate MLP's hidden pre-activation W3 msg + b3 =
    // (W3 W2) a1 + (W3 b2 + b3) are both linear in a1: the stacked panel [W2 ; W3 W2] gives them from one A operand
    // (no bf16x3 split of msg), as two N=64 halves.
    {
      auto w23 = [&](int hn) {
        return [&, hn](int sp, int kb) {
          return b_desc_ex(w_saddr + TC_W23_BASE + sp * TC_W23_SPLIT + kb * 4096 + hn * 1024, 2048, 128); };
      };
      float m[32], hd[32];
      wg_gemm6_rs_issue<64, 4, 0, false, P>(m, af, w23(0), false);
      wg_gemm6_rs_issue<64, 4, 0, false, P>(hd, af, w23(1), false);
      wg_mma_wait(m);
      wg_mma_wait(hd);   // (the second wait only pins hd behind the first)
      float u[32];   // LeakyReLU(hidden + b3)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float2 b2 = *reinterpret_cast<const float2*>(&cst.b2[8 * j + fc]);
        const float2 b3 = *reinterpret_cast<const float2*>(&cst.b3[8 * j + fc]);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          *reinterpret_cast<float2*>(W.msg + (fr0 + 8 * h) * TC_LD + 8 * j + fc) =
              make_float2(__fadd_rn(m[4 * j + 2 * h], b2.x), __fadd_rn(m[4 * j + 2 * h + 1], b2.y));
          const float x0 = __fadd_rn(hd[4 * j + 2 * h], b3.x), x1 = __fadd_rn(hd[4 * j + 2 * h + 1], b3.y);
          u[4 * j + 2 * h] = fmaxf(x0, __fmul_rn(x0, slope));
          u[4 * j + 2 * h + 1] = fmaxf(x1, __fmul_rn(x1, slope));
        }
      }
      if (CLN) {   // coors_mlp.3
        float mean[2], rstd[2];
        quad_ln_stats(u, mean, rstd);
        quad_ln_apply(u, mean, rstd, cln, cln + 64, fc);
      }
      // phi = w4 . u + b_coor2 in the chain order of the row-per-thread formulation: four fp32 chains per 32-column half,
      // combined in fp64
      float pu[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) pu[i] = __shfl_xor_sync(0xffffffffu, u[i], 2);
      double phv[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        double red[2];
#pragma unroll
        for (int ch = 0; ch < 2; ++ch) {
          const float* w4 = cst.w4 + 32 * ch + 2 * (lane & 1);
          float p0 = 0.f, p1 = 0.f;
#pragma unroll
          for (int c4 = 0; c4 < 8; ++c4) {
            p0 = fmaf(chain_val(u, pu, h, ch, c4, 0), w4[4 * c4], p0);
            p1 = fmaf(chain_val(u, pu, h, ch, c4, 1), w4[4 * c4 + 1], p1);
          }
          const double pp = (double)p0 + (double)p1;
          red[ch] = pp + __shfl_xor_sync(0xffffffffu, pp, 1);
        }
        phv[h] = red[0] + red[1] + (double)p.b_coor2;
      }
      if ((lane & 3) == 0) {
        W.phi[fr0] = phv[0];
        W.phi[fr0 + 8] = phv[1];
      }
    }
    wg_barrier(bar);   // msg tile, phi and x_rel complete
    // ---- coordinate update :264, 274-277, 286-292 on the last threads ------------------------------------------------
    if (o_upd < nn * 3) {
      const int rs = W.rp[buf][nd_upd] - e0, re = W.rp[buf][nd_upd + 1] - e0;
      double sum = 0.0;
      if (deg10) {   // fixed in-degree: the same fused multiply-add chain, unrolled (its shared loads go out together)
#pragma unroll
        for (int j = 0; j < 10; ++j) {
          const int rr = nd_upd * 10 + j;
          sum += W.xm[rr * 3 + comp_upd] * W.phi[rr];
        }
      } else {
        for (int rr = rs; rr < re; ++rr) sum += W.xm[rr * 3 + comp_upd] * W.phi[rr];  // x_rel * phi :264
      }
      const int deg = re - rs;
      const double upd = deg > 0 ? sum / (double)deg : 0.0;
      const double eta = (double)p.x_connection_init;
      x_out[gi_upd] = eta * xo_upd + (1.0 - eta) * xi_upd + upd;
    }
    // ---- mean aggregation of msg at the destination nodes (:280-283): 2 threads per channel, each a run of nodes -------
    {
      const int c = t & 63;
      const float* col = W.msg + c;
      if (deg10) {  // same sums, no row_ptr lookups
        for (int nd = (nn * half) >> 1, nd1 = (nn * (half + 1)) >> 1; nd < nd1; ++nd) {
          const float* cr = col + nd * 10 * TC_LD;
          float s0 = 0.f, s1 = 0.f;
#pragma unroll
          for (int j = 0; j < 10; j += 2) {
            s0 += cr[j * TC_LD];
            s1 += cr[(j + 1) * TC_LD];
          }
          aggr[(long)(n0 + nd) * 64 + c] = (s0 + s1) / 10.f;
        }
      } else {
        for (int nd = (nn * half) >> 1, nd1 = (nn * (half + 1)) >> 1; nd < nd1; ++nd) {
          const int rs = W.rp[buf][nd] - e0, re = W.rp[buf][nd + 1] - e0;
          float s0 = 0.f, s1 = 0.f;
          int rr = rs;
          for (; rr + 1 < re; rr += 2) {
            s0 += col[rr * TC_LD];
            s1 += col[(rr + 1) * TC_LD];
          }
          if (rr < re) s0 += col[rr * TC_LD];
          aggr[(long)(n0 + nd) * 64 + c] = re > rs ? (s0 + s1) / (float)(re - rs) : 0.f;
        }
      }
    }
    e0 = e0n; ne = nen; off_l = off_ln; n_l = n_ln; off_r = off_rn; buf ^= 1;
  }
  cp_async_wait<0>();
  __syncthreads();
}

template <int P, bool CLN>
static int launch_edge_stage_tc(const eqd_graph* g, const eqd_layer* p_l, const float* proj, const double* x_in,
                                const double* x_orig, float* aggr, double* x_out, int32_t* status, int tn, void* stream) {
  const int ntiles = (g->n_nodes + tn - 1) / tn;
  EdgeConsts cst;
  memcpy(&cst, p_l->consts.edge, sizeof(cst));
  size_t smem = sizeof(TcSmem) + 128 + (CLN ? TC_CLN_BYTES : 0);
  EQD_SET_SMEM((edge_stage_tc_kernel<P, CLN>), smem);
  int grid = (ntiles + TC_WGS - 1) / TC_WGS;
  if (grid > EQD_SMS) grid = EQD_SMS;
  edge_stage_tc_kernel<P, CLN><<<grid, TC_THREADS, smem, (cudaStream_t)stream>>>(*g, p_l->dev, cst, proj, x_in, x_orig,
                                                                                aggr, x_out, status, tn, p_l->norms);
  EQD_CUDA_LAUNCH_CHECK();
  return EQD_OK;
}

}  // namespace eqd

extern "C" int eqd_edge_stage(const eqd_graph* g, const eqd_layer* p_l, const float* proj, const double* x_in,
                              const double* x_orig, float* aggr, double* x_out, int32_t* status, void* stream) {
  const eqd_layer_params* p = p_l ? &p_l->dev : nullptr;
  if (!g || !p || !proj || !x_in || !x_orig || !aggr || !x_out || !status) return EQD_ERR_BAD_ARG;
  if (!p->w_edge_tc) return EQD_ERR_BAD_ARG;
  const int cln = eqd_coors_ln(p_l);
  if (cln < 0) return EQD_ERR_BAD_ARG;
  const int products = eqd_mma_products(p);
  if (!products) return EQD_ERR_UNSUPPORTED;
  if (g->max_in_degree < 1 || g->max_in_degree > EQD_TM) return EQD_ERR_UNSUPPORTED;
  if (!(p->leaky_slope >= 0.f && p->leaky_slope <= 1.f)) return EQD_ERR_UNSUPPORTED;  // lrelu() = max(v, slope*v)
  if ((reinterpret_cast<uintptr_t>(g->he_lig) | reinterpret_cast<uintptr_t>(g->he_rec) |
       reinterpret_cast<uintptr_t>(p->w_edge_tc)) & 15)
    return EQD_ERR_BAD_ARG;  // bulk copies need 16-byte aligned bases
  // a node's in-edges must fit one 64-row warpgroup tile; larger bounds, and training-mode dropout, run on the fp32 kernel
  if (g->max_in_degree > TC_ROWS || p_l->dropout.p > 0.f) return eqd_edge_stage_ffma(g, p_l, proj, x_in, x_orig, aggr, x_out, status, stream);
  if (g->n_nodes <= 0) return EQD_OK;
  int tn = TC_ROWS / g->max_in_degree;
  if (tn > TC_MAX_TN) tn = TC_MAX_TN;
  if (cln)
    return products == 3 ? eqd::launch_edge_stage_tc<3, true>(g, p_l, proj, x_in, x_orig, aggr, x_out, status, tn, stream)
                         : eqd::launch_edge_stage_tc<6, true>(g, p_l, proj, x_in, x_orig, aggr, x_out, status, tn, stream);
  return products == 3 ? eqd::launch_edge_stage_tc<3, false>(g, p_l, proj, x_in, x_orig, aggr, x_out, status, tn, stream)
                       : eqd::launch_edge_stage_tc<6, false>(g, p_l, proj, x_in, x_orig, aggr, x_out, status, tn, stream);
}
