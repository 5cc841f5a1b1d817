// Shared device helpers for the IEGMN forward kernels (sm_90a).
//
// Tile model used by every dense stage: one CTA = 128 threads owns a tile of 128 rows (edges or
// nodes) x 64 output channels.  Thread (ty = tid>>3, tx = tid&7) holds an 8x8 fp32 micro-tile:
//   rows  ty*8 + i                      i = 0..7
//   cols  tx*4 + (j&3) + 32*(j>>2)      j = 0..7      ("NN" GEMMs, W k-major)
//   cols  tx + 8*j                      j = 0..7      ("NT" GEMM,  S = Q K^T)
// plus, for the 69(72)-wide layer-0 tensors, one extra column 64+tx ("EXTRA").
// The A operand lives in shared memory row-major with a padded row stride (multiple of 4 floats)
// so a quarter-warp reads one 16-byte word (broadcast); the W operand is k-major so a quarter-warp
// reads 128 contiguous bytes: both conflict-free, 16 FFMA per LDS.128.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/eqd_iegmn.h"

#define EQD_THREADS 128
#define EQD_TM 128
// streaming multiprocessors of an H100 SXM: the grid size of the persistent kernels
#define EQD_SMS 132

#define EQD_CUDA_LAUNCH_CHECK()                          \
  do {                                                   \
    cudaError_t e__ = cudaGetLastError();                \
    if (e__ != cudaSuccess) return -(1000 + (int)e__);   \
  } while (0)

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) once per (call site = kernel instantiation, device) instead of on
// every launch; re-issued only if a larger size is ever requested.  A benign race between host threads at worst sets
// the same value twice.
#define EQD_SET_SMEM(kernel, bytes)                                                                            \
  do {                                                                                                         \
    static int eqd_smem_set_[64];                                                                              \
    int dev__ = 0;                                                                                             \
    cudaGetDevice(&dev__);                                                                                     \
    if (dev__ < 0 || dev__ >= 64 || eqd_smem_set_[dev__] < (int)(bytes)) {                                     \
      cudaError_t e__ = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(bytes)); \
      if (e__ != cudaSuccess) return -(1000 + (int)e__);                                                       \
      if (dev__ >= 0 && dev__ < 64) eqd_smem_set_[dev__] = (int)(bytes);                                       \
    }                                                                                                          \
  } while (0)

// Product count of a layer's tensor-core GEMMs (eqd_layer_params.mma_products): 6 for 0 or 6 (bf16x6), 3 for 3 on a
// 64-wide layer (bf16x3); 0 for any other value, which the tensor-core launchers refuse with EQD_ERR_UNSUPPORTED.
inline int eqd_mma_products(const eqd_layer_params* p) {
  if (p->mma_products == 0 || p->mma_products == 6) return 6;
  return p->mma_products == 3 && p->dh == EQD_HID ? 3 : 0;
}

namespace eqd {

// LeakyReLU for 0 <= slope <= 1 (checked by the launchers): max(v, slope*v) is bit-identical to the select form
// and one instruction shorter (FMUL + FMNMX)
__device__ __forceinline__ float lrelu(float v, float slope) { return fmaxf(v, v * slope); }

__device__ __forceinline__ int col_nn(int tx, int j) { return tx * 4 + (j & 3) + ((j >> 2) << 5); }
__device__ __forceinline__ int col_nt(int tx, int j) { return tx + 8 * j; }

__device__ __forceinline__ float f4_get(const float4& v, int k) {
  return k == 0 ? v.x : (k == 1 ? v.y : (k == 2 ? v.z : v.w));
}

// ---- cp.async (LDGSTS) helpers ---------------------------------------------------------------
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src, bool valid) {
  unsigned dst = (unsigned)__cvta_generic_to_shared(smem_dst);
  int src_bytes = valid ? 16 : 0;  // src-size 0 => zero fill
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(dst), "l"(gmem_src), "r"(src_bytes));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

// Copy `nrows` rows of `ncols` floats (ncols % 4 == 0) from global (row stride ld_g) into shared
// memory (row stride ld_s).  Rows >= nvalid are zero-filled.  Asynchronous: caller commits/waits.
__device__ __forceinline__ void tile_load_async(float* __restrict__ dst, int ld_s, const float* __restrict__ src,
                                                long ld_g, int nrows, int nvalid, int ncols, int tid) {
  const int c4n = ncols >> 2;
  const int total = nrows * c4n;
  for (int idx = tid; idx < total; idx += EQD_THREADS) {
    int r = idx / c4n, c4 = idx - r * c4n;
    bool ok = r < nvalid;
    const float* s = src + (ok ? (long)r * ld_g + c4 * 4 : 0);
    cp_async16(dst + r * ld_s + c4 * 4, s, ok);
  }
}

// ---- GEMM micro-kernels -----------------------------------------------------------------------
// acc[i][j] += sum_k A[i][k] * W[k][col_nn(j)],  A: smem pointer to this thread's first row.
template <bool EXTRA>
__device__ __forceinline__ void gemm_nn(float (&acc)[8][8], float (&accx)[8], const float* __restrict__ A, int lda,
                                        const float* __restrict__ W, int ldw, int K, int tx) {
  const float* wp = W + tx * 4;
#pragma unroll 1
  for (int k = 0; k < K; k += 4) {
    float4 av[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) av[i] = *reinterpret_cast<const float4*>(A + i * lda + k);
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      const float* wr = wp + (k + kk) * ldw;
      float4 w0 = *reinterpret_cast<const float4*>(wr);
      float4 w1 = *reinterpret_cast<const float4*>(wr + 32);
      float wx = 0.f;
      if (EXTRA) wx = W[(k + kk) * ldw + 64 + tx];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float a = f4_get(av[i], kk);
        acc[i][0] = fmaf(a, w0.x, acc[i][0]);
        acc[i][1] = fmaf(a, w0.y, acc[i][1]);
        acc[i][2] = fmaf(a, w0.z, acc[i][2]);
        acc[i][3] = fmaf(a, w0.w, acc[i][3]);
        acc[i][4] = fmaf(a, w1.x, acc[i][4]);
        acc[i][5] = fmaf(a, w1.y, acc[i][5]);
        acc[i][6] = fmaf(a, w1.z, acc[i][6]);
        acc[i][7] = fmaf(a, w1.w, acc[i][7]);
        if (EXTRA) accx[i] = fmaf(a, wx, accx[i]);
      }
    }
  }
}

// acc[i][j] += sum_k A[i][k] * B[col_nt(j)][k]   (both operands row-major in smem, K % 4 == 0)
__device__ __forceinline__ void gemm_nt(float (&acc)[8][8], const float* __restrict__ A, int lda,
                                        const float* __restrict__ B, int ldb, int K, int tx) {
  const float* bp = B + tx * ldb;
#pragma unroll 1
  for (int k = 0; k < K; k += 4) {
    float4 av[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) av[i] = *reinterpret_cast<const float4*>(A + i * lda + k);
#pragma unroll
    for (int jh = 0; jh < 2; ++jh) {
      float4 bv[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) bv[j] = *reinterpret_cast<const float4*>(bp + (jh * 4 + j) * 8 * ldb + k);
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          float a = f4_get(av[i], kk);
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][jh * 4 + j] = fmaf(a, f4_get(bv[j], kk), acc[i][jh * 4 + j]);
        }
    }
  }
}

// Streams a k-major weight panel W[K][ncols] (global / L2, row stride ldw_g floats) through a
// double-buffered shared-memory ring of 32-row chunks and accumulates acc += A . W.
// wbuf: 2 * 32 * WLD floats, WLD = 72.  All 128 threads must call it (contains __syncthreads).
#define EQD_WCHUNK 32
#define EQD_WLD 72
template <bool EXTRA>
__device__ __forceinline__ void gemm_nn_stream(float (&acc)[8][8], float (&accx)[8], const float* __restrict__ A,
                                               int lda, int K, const float* __restrict__ Wg, int ldw_g, int ncols,
                                               float* __restrict__ wbuf, int tid) {
  const int tx = tid & 7;
  const int c4n = ncols >> 2;
  const int nchunks = (K + EQD_WCHUNK - 1) / EQD_WCHUNK;
  auto issue = [&](int c) {
    float* dst = wbuf + (c & 1) * (EQD_WCHUNK * EQD_WLD);
    int k0 = c * EQD_WCHUNK;
    int rows = min(EQD_WCHUNK, K - k0);
    int total = rows * c4n;
    for (int idx = tid; idx < total; idx += EQD_THREADS) {
      int r = idx / c4n, c4 = idx - r * c4n;
      cp_async16(dst + r * EQD_WLD + c4 * 4, Wg + (long)(k0 + r) * ldw_g + c4 * 4, true);
    }
    cp_async_commit();
  };
  issue(0);
  for (int c = 0; c < nchunks; ++c) {
    if (c + 1 < nchunks) {
      issue(c + 1);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    int k0 = c * EQD_WCHUNK;
    int rows = min(EQD_WCHUNK, K - k0);
    gemm_nn<EXTRA>(acc, accx, A + k0, lda, wbuf + (c & 1) * (EQD_WCHUNK * EQD_WLD), EQD_WLD, rows, tx);
    __syncthreads();
  }
}

// ---- row-wise reductions over the 8 lanes (tx) that share a row ---------------------------------
__device__ __forceinline__ float row_sum8(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  v += __shfl_xor_sync(0xffffffffu, v, 2);
  v += __shfl_xor_sync(0xffffffffu, v, 4);
  return v;
}
__device__ __forceinline__ float row_max8(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 4));
  return v;
}

// LeakyReLU then nn.LayerNorm (biased variance, eps 1e-5) over `dh` real channels of each row.
// EXTRA: channels 64..64+7 live in accx (valid iff 64+tx < dh).  gamma/beta indexed by channel.
template <bool EXTRA>
__device__ __forceinline__ void lrelu_layernorm(float (&acc)[8][8], float (&accx)[8], const float* __restrict__ gamma,
                                                const float* __restrict__ beta, int dh, float slope, int tx) {
  const float inv_n = 1.f / (float)dh;
  const bool xvalid = EXTRA && (64 + tx < dh);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      acc[i][j] = lrelu(acc[i][j], slope);
      s += acc[i][j];
    }
    if (EXTRA) {
      accx[i] = xvalid ? lrelu(accx[i], slope) : 0.f;
      s += accx[i];
    }
    float mean = row_sum8(s) * inv_n;
    float q = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float d = acc[i][j] - mean;
      q = fmaf(d, d, q);
    }
    if (EXTRA && xvalid) {
      float d = accx[i] - mean;
      q = fmaf(d, d, q);
    }
    float var = row_sum8(q) * inv_n;
    float rstd = 1.f / sqrtf(var + 1e-5f);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      int c = col_nn(tx, j);
      acc[i][j] = (acc[i][j] - mean) * rstd * gamma[c] + beta[c];
    }
    if (EXTRA) accx[i] = xvalid ? (accx[i] - mean) * rstd * gamma[64 + tx] + beta[64 + tx] : 0.f;
  }
}

// Store the micro-tile (NN column map) row-major into shared memory (row stride ld).
template <bool EXTRA>
__device__ __forceinline__ void store_tile_smem(float* __restrict__ S, int ld, const float (&acc)[8][8],
                                                const float (&accx)[8], int ty, int tx) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    float* r = S + (ty * 8 + i) * ld + tx * 4;
    *reinterpret_cast<float4*>(r) = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
    *reinterpret_cast<float4*>(r + 32) = make_float4(acc[i][4], acc[i][5], acc[i][6], acc[i][7]);
    if (EXTRA) S[(ty * 8 + i) * ld + 64 + tx] = accx[i];
  }
}

__device__ __forceinline__ void acc_set_bias(float (&acc)[8][8], const float* __restrict__ bias, int tx) {
  float b[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) b[j] = bias ? bias[col_nn(tx, j)] : 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = b[j];
}

// Project a 128-row tile held in shared memory (A, K = dhp_in columns) through the projection
// panel of layer `p` (see eqd_layer_params.w_proj) and write proj[node][128 + 3*dhp].
// Used by the standalone projection kernel (layer 0) and fused into the node stage.
template <bool EXTRA>
__device__ __forceinline__ void project_tile(const float* __restrict__ A, int lda, const eqd_layer_params& p,
                                             float* __restrict__ proj, int node0, int nvalid, float* wbuf, int tid) {
  const int ty = tid >> 3, tx = tid & 7;
  const int dhp = p.dhp;
  const int pw = 128 + 3 * dhp;
#pragma unroll 1
  for (int g = 0; g < 5; ++g) {
    const int off = g < 2 ? g * 64 : 128 + (g - 2) * dhp;
    const bool ex = EXTRA && g >= 2;
    float acc[8][8], accx[8];
    acc_set_bias(acc, p.b_proj + off, tx);
#pragma unroll
    for (int i = 0; i < 8; ++i) accx[i] = ex ? p.b_proj[off + 64 + tx] : 0.f;
    if (ex)
      gemm_nn_stream<true>(acc, accx, A + ty * 8 * lda, lda, dhp, p.w_proj + off, pw, 72, wbuf, tid);
    else
      gemm_nn_stream<false>(acc, accx, A + ty * 8 * lda, lda, dhp, p.w_proj + off, pw, 64, wbuf, tid);
    const bool act = (g == 2 || g == 3);  // Q, K carry the LeakyReLU; Psrc/Pdst/V are linear
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      int r = ty * 8 + i;
      if (r < nvalid) {
        float v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = act ? lrelu(acc[i][j], p.leaky_slope) : acc[i][j];
        float* o = proj + (long)(node0 + r) * pw + off + tx * 4;
        *reinterpret_cast<float4*>(o) = make_float4(v[0], v[1], v[2], v[3]);
        *reinterpret_cast<float4*>(o + 32) = make_float4(v[4], v[5], v[6], v[7]);
        if (ex) proj[(long)(node0 + r) * pw + off + 64 + tx] = act ? lrelu(accx[i], p.leaky_slope) : accx[i];
      }
    }
  }
}

}  // namespace eqd
