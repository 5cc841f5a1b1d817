// Shared helpers of the BACKWARD kernels (bwd_*.cu).  The backward of the IEGMN path has no code in the reference: it is
// what torch.autograd makes of rigid_docking_model.py (`loss.backward()`, src/train.py:154).  The chain rule implemented
// here is restated, stage by stage and with the same stage boundaries, in oracle/backward_manual.py (pinned against
// torch.autograd and the reference's own golden gradients).
//
// Design: fp32 FFMA tile kernels (128 threads, 128-row tiles, the 8x8 micro-tile machinery of common.cuh) recompute the
// per-edge / per-node activations from the stashed layer inputs and produce the DATA gradients; every WEIGHT gradient is
// a row reduction  dW[k][n] = sum_rows X[row][k] * D[row][n]  over operand matrices the tile kernels leave in HBM, done
// by ONE generic kernel (tn_gemm_kernel: per-row-chunk partials) followed by a deterministic fixed-order second stage
// (grad_reduce_kernel) that also scatters the packed k-major panels into the flat parameter-gradient buffer.  No float
// atomics anywhere: gradients are bit-reproducible for a given batch.
#pragma once
#include "common.cuh"

namespace eqd {

// d leaky_relu / d pre, PyTorch convention: pre > 0 ? 1 : slope.  `post` = lrelu(pre): same sign as pre for slope > 0,
// and post == 0 exactly when pre <= 0 for slope == 0.
__device__ __forceinline__ float lrelu_grad_from_post(float post, float slope) { return post > 0.f ? 1.f : slope; }

// nn.LayerNorm backward of one row held by its 8 lanes: dnh = dL/d(output) * gamma and nhat = the normalised input at
// this lane's 8 columns (with EXTRA also column 64 + tx in dnhx / nhx, 0 for a column past the row's width), rstd of the
// row (ln_row_stats), inv_n = 1 / channel count.  Overwrites dnh (dnhx) with dL/d(input) = rstd (dnh - m1 - nhat m2),
// m1 = mean(dnh), m2 = mean(dnh nhat); the caller multiplies in the activation's derivative afterwards.
template <bool EXTRA>
__device__ __forceinline__ void layernorm_bwd_row(float (&dnh)[8], float& dnhx, const float (&nhat)[8], float nhx,
                                                  float rstd, float inv_n) {
  float s1 = 0.f, s2 = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    s1 += dnh[j];
    s2 = fmaf(dnh[j], nhat[j], s2);
  }
  if (EXTRA) {
    s1 += dnhx;
    s2 = fmaf(dnhx, nhx, s2);
  }
  const float m1 = row_sum8(s1) * inv_n, m2 = row_sum8(s2) * inv_n;
#pragma unroll
  for (int j = 0; j < 8; ++j) dnh[j] = rstd * (dnh[j] - m1 - nhat[j] * m2);
  if (EXTRA) dnhx = rstd * (dnhx - m1 - nhx * m2);
}
// The same for a 64-wide row.
__device__ __forceinline__ void layernorm_bwd_row(float (&dnh)[8], const float (&nhat)[8], float rstd) {
  float unused = 0.f;
  layernorm_bwd_row<false>(dnh, unused, nhat, 0.f, rstd, 1.f / 64.f);
}

// Adds this thread's 8 rows of an 8x8 micro-tile into per-thread column accumulators (column map col_nn).
__device__ __forceinline__ void colacc8(float (&s)[8], const float (&v)[8][8]) {
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += v[i][j];
    s[j] += t;
  }
}

// Per-CTA reduction of per-thread column accumulators over the 16 row groups (ty), in fixed order, written to
// out[col_nn(tx, j)].  scratch: 16 * 64 floats.  All 128 threads call it (contains __syncthreads).
__device__ __forceinline__ void colacc8_flush(const float (&s)[8], float* scratch, float* __restrict__ out, int tid) {
  const int ty = tid >> 3, tx = tid & 7;
  __syncthreads();
#pragma unroll
  for (int j = 0; j < 8; ++j) scratch[ty * 64 + col_nn(tx, j)] = s[j];
  __syncthreads();
  if (tid < 64) {
    float t = 0.f;
#pragma unroll
    for (int q = 0; q < 16; ++q) t += scratch[q * 64 + tid];
    out[tid] = t;
  }
  __syncthreads();
}

// Writes this thread's rows of a 128 x 64 micro-tile (col_nn map) to a row-major global matrix (row stride ld floats).
__device__ __forceinline__ void store_tile_global(float* __restrict__ G, long row0, int ld, int nvalid,
                                                  const float (&acc)[8][8], int ty, int tx) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    int r = ty * 8 + i;
    if (r < nvalid) {
      float* o = G + (row0 + r) * ld + tx * 4;
      *reinterpret_cast<float4*>(o) = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
      *reinterpret_cast<float4*>(o + 32) = make_float4(acc[i][4], acc[i][5], acc[i][6], acc[i][7]);
    }
  }
}

}  // namespace eqd
