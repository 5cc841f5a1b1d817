// Weight-gradient machinery of the backward pass: the generic row-reduction GEMM, the deterministic second stage that
// scatters packed partials into the flat parameter-gradient buffer, and the optimiser-side kernels that run on that flat
// buffer (squared-norm partials for clip_grad_norm_, fused clip + Adam; src/train.py:156, 165, 302).
#include "bwd_common.cuh"

namespace eqd {

#define TN_ROWS 64   // rows per smem sub-tile
#define TN_LD 68

// partial[chunk][k][n] = alpha * sum_{r in chunk} X[r][k] * D[r][n]      (k < K, n < ncols)
// colsum[chunk][n]     = alpha * sum_{r in chunk} D[r][n]                (optional, written by the kb == 0 CTAs)
// grid = (nchunks, kblocks * nblocks); one CTA = one 64 x 64 output block over one row chunk.
__global__ void __launch_bounds__(EQD_THREADS)
tn_gemm_kernel(const float* __restrict__ X, int ldx, int K, const float* __restrict__ D, int ldd, int ncols, long nrows,
               int rows_per_chunk, float alpha, float* __restrict__ partial, float* __restrict__ colsum) {
  extern __shared__ __align__(16) float smem[];
  float* Xs = smem;                          // [2][TN_ROWS][TN_LD]
  float* Ds = smem + 2 * TN_ROWS * TN_LD;    // [2][TN_ROWS][TN_LD]
  const int tid = threadIdx.x, ty = tid >> 3, tx = tid & 7;
  const int nblocks = (ncols + 63) / 64;
  const int kb = blockIdx.y / nblocks, nb = blockIdx.y - kb * nblocks;
  const int k0 = kb * 64, n0 = nb * 64;
  const int kw = min(64, K - k0), nw = min(64, ncols - n0);   // valid widths (multiples of 4)
  const long r_begin = (long)blockIdx.x * rows_per_chunk;
  const long r_end = min(nrows, r_begin + rows_per_chunk);
  const bool do_colsum = colsum != nullptr && kb == 0;

  auto issue = [&](int buf, long r0) {
    const int nv = (int)min((long)TN_ROWS, r_end - r0);
    float* xd = Xs + buf * TN_ROWS * TN_LD;
    float* dd = Ds + buf * TN_ROWS * TN_LD;
    for (int idx = tid; idx < TN_ROWS * 16; idx += EQD_THREADS) {
      int r = idx >> 4, c4 = idx & 15;
      bool okx = r < nv && c4 * 4 < kw, okd = r < nv && c4 * 4 < nw;
      cp_async16(xd + r * TN_LD + c4 * 4, X + (okx ? (r0 + r) * ldx + k0 + c4 * 4 : 0), okx);
      cp_async16(dd + r * TN_LD + c4 * 4, D + (okd ? (r0 + r) * ldd + n0 + c4 * 4 : 0), okd);
    }
    cp_async_commit();
  };

  float acc[4][8], cs[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    cs[j] = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) acc[i][j] = 0.f;
  }
  int buf = 0;
  if (r_begin < r_end) issue(0, r_begin);
  for (long r0 = r_begin; r0 < r_end; r0 += TN_ROWS) {
    if (r0 + TN_ROWS < r_end) {
      issue(buf ^ 1, r0 + TN_ROWS);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    const float* xs = Xs + buf * TN_ROWS * TN_LD + ty * 4;
    const float* ds = Ds + buf * TN_ROWS * TN_LD + tx * 4;
#pragma unroll 4
    for (int r = 0; r < TN_ROWS; ++r) {     // rows past the chunk end were zero-filled
      float4 a = *reinterpret_cast<const float4*>(xs + r * TN_LD);
      float4 d0 = *reinterpret_cast<const float4*>(ds + r * TN_LD);
      float4 d1 = *reinterpret_cast<const float4*>(ds + r * TN_LD + 32);
      const float av[4] = {a.x, a.y, a.z, a.w};
      const float dv[8] = {d0.x, d0.y, d0.z, d0.w, d1.x, d1.y, d1.z, d1.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(av[i], dv[j], acc[i][j]);
      if (do_colsum && (r & 15) == ty) {
#pragma unroll
        for (int j = 0; j < 8; ++j) cs[j] += dv[j];
      }
    }
    __syncthreads();
    buf ^= 1;
  }
  float* out = partial + (long)blockIdx.x * K * ncols;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    int k = k0 + ty * 4 + i;
    if (k < K) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        int n = n0 + col_nn(tx, j);
        if (n < ncols) out[(long)k * ncols + n] = alpha * acc[i][j];
      }
    }
  }
  if (do_colsum) {   // fixed-order reduction over the 16 row groups
    float* scratch = smem;
#pragma unroll
    for (int j = 0; j < 8; ++j) scratch[ty * 64 + col_nn(tx, j)] = cs[j];
    __syncthreads();
    if (tid < 64 && n0 + tid < ncols) {
      float t = 0.f;
#pragma unroll
      for (int q = 0; q < 16; ++q) t += scratch[q * 64 + tid];
      colsum[(long)blockIdx.x * ncols + n0 + tid] = alpha * t;
    }
  }
}

// grad[dst[i]] += sum_c partial[c * stride + src[i]]   (fixed order over c, fp64 accumulation): the deterministic second
// stage of every weight gradient, and the scatter from the kernels' packed layouts to the state_dict layout.
__global__ void grad_reduce_kernel(const float* __restrict__ partial, int nchunks, long stride, const int* __restrict__ src,
                                   const int* __restrict__ dst, int n, float* __restrict__ grad) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* p = partial + src[i];
  double t = 0.0;
  for (int c = 0; c < nchunks; ++c) t += (double)p[(long)c * stride];
  grad[dst[i]] += (float)t;
}

// ---- optimiser side, on the flat gradient buffer -------------------------------------------------------------------
// partial[b] = sum of squares of this block's slice (fixed order inside the block: per-thread strided sums, then a tree).
__global__ void sqnorm_partial_kernel(const float* __restrict__ g, long n, double* __restrict__ partial) {
  __shared__ double sh[256];
  long per = (n + gridDim.x - 1) / gridDim.x;
  long lo = (long)blockIdx.x * per, hi = min(n, lo + per);
  double t = 0.0;
  for (long i = lo + threadIdx.x; i < hi; i += blockDim.x) t += (double)g[i] * (double)g[i];
  sh[threadIdx.x] = t;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) partial[blockIdx.x] = sh[0];
}

// clip_grad_norm_(max_norm) (train.py:156) fused with torch.optim.Adam's step (train.py:165, 302; weight_decay = L2 added
// to the gradient, no amsgrad): the global norm is the sqrt of the sum of `n_partial` doubles; `scale_extra` multiplies
// the gradient first (1 / world for an averaged all-reduce).  One pass over the flat buffers.
__global__ void clip_adam_kernel(float* __restrict__ w, float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                                 long n, const double* __restrict__ sq_partial, int n_partial, float max_norm,
                                 float lr, float beta1, float beta2, float eps, float weight_decay, float bc1, float bc2,
                                 float scale_extra, float* __restrict__ norm_out) {
  double tot = 0.0;
  for (int i = 0; i < n_partial; ++i) tot += sq_partial[i];
  const float norm = (float)sqrt(tot) * fabsf(scale_extra);
  float clip = max_norm / (norm + 1e-6f);     // torch.nn.utils.clip_grad_norm_: clip_coef clamped to 1
  clip = clip < 1.f ? clip : 1.f;
  if (norm_out && blockIdx.x == 0 && threadIdx.x == 0) *norm_out = norm;
  long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float gi = g[i] * scale_extra * clip;
  g[i] = gi;
  if (weight_decay != 0.f) gi = fmaf(weight_decay, w[i], gi);
  float mi = beta1 * m[i] + (1.f - beta1) * gi;
  float vi = beta2 * v[i] + (1.f - beta2) * gi * gi;
  m[i] = mi;
  v[i] = vi;
  float denom = sqrtf(vi) / sqrtf(bc2) + eps;
  w[i] -= (lr / bc1) * (mi / denom);
}

}  // namespace eqd

extern "C" size_t eqd_tn_partial_floats(int64_t nrows, int32_t K, int32_t ncols, int32_t* rows_per_chunk_out,
                                        int32_t* nchunks_out) {
  if (nrows <= 0 || K <= 0 || ncols <= 0) {
    if (rows_per_chunk_out) *rows_per_chunk_out = 0;
    if (nchunks_out) *nchunks_out = 0;
    return 0;
  }
  const int blocks = ((K + 63) / 64) * ((ncols + 63) / 64);
  long target = (EQD_SMS * 4 + blocks - 1) / blocks;               // ~4 CTAs per SM over the whole launch
  long rpc = (nrows + target - 1) / target;
  rpc = ((rpc + 63) / 64) * 64;
  if (rpc < 256) rpc = 256;
  long nch = (nrows + rpc - 1) / rpc;
  if (rows_per_chunk_out) *rows_per_chunk_out = (int32_t)rpc;
  if (nchunks_out) *nchunks_out = (int32_t)nch;
  return (size_t)nch * (size_t)K * (size_t)ncols;
}

extern "C" int eqd_tn_gemm(const float* X, int32_t ldx, int32_t K, const float* D, int32_t ldd, int32_t ncols,
                           int64_t nrows, float alpha, float* partial, float* colsum, int32_t* nchunks_out,
                           void* stream) {
  if (!X || !D || !partial || K <= 0 || ncols <= 0 || (K & 3) || (ncols & 3) || (ldx & 3) || (ldd & 3))
    return EQD_ERR_BAD_ARG;
  if ((reinterpret_cast<uintptr_t>(X) | reinterpret_cast<uintptr_t>(D)) & 15) return EQD_ERR_BAD_ARG;
  int32_t rpc = 0, nch = 0;
  eqd_tn_partial_floats(nrows, K, ncols, &rpc, &nch);
  if (nchunks_out) *nchunks_out = nch;
  if (nrows <= 0) return EQD_OK;
  size_t smem = (size_t)4 * TN_ROWS * TN_LD * sizeof(float);
  EQD_SET_SMEM((eqd::tn_gemm_kernel), smem);
  dim3 grid((unsigned)nch, (unsigned)(((K + 63) / 64) * ((ncols + 63) / 64)));
  eqd::tn_gemm_kernel<<<grid, EQD_THREADS, smem, (cudaStream_t)stream>>>(X, ldx, K, D, ldd, ncols, nrows, rpc, alpha,
                                                                        partial, colsum);
  EQD_CUDA_LAUNCH_CHECK();
  return EQD_OK;
}

extern "C" int eqd_grad_reduce(const float* partial, int32_t nchunks, int64_t stride, const int32_t* src_index,
                               const int32_t* dst_index, int32_t n, float* grad, void* stream) {
  if (!partial || !src_index || !dst_index || !grad || nchunks < 0 || n < 0) return EQD_ERR_BAD_ARG;
  if (n == 0 || nchunks == 0) return EQD_OK;
  eqd::grad_reduce_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(partial, nchunks, stride, src_index,
                                                                             dst_index, n, grad);
  EQD_CUDA_LAUNCH_CHECK();
  return EQD_OK;
}

extern "C" int eqd_sqnorm_partials(const float* g, int64_t n, double* partial, int32_t n_partial, void* stream) {
  if (!g || !partial || n < 0 || n_partial <= 0 || n_partial > 1024) return EQD_ERR_BAD_ARG;
  eqd::sqnorm_partial_kernel<<<n_partial, 256, 0, (cudaStream_t)stream>>>(g, n, partial);
  EQD_CUDA_LAUNCH_CHECK();
  return EQD_OK;
}

extern "C" int eqd_clip_adam(float* w, float* g, float* m, float* v, int64_t n, const double* sq_partial,
                             int32_t n_partial, float max_norm, float lr, float beta1, float beta2, float eps,
                             float weight_decay, int32_t step, float scale_extra, float* norm_out, void* stream) {
  // the partial count is that of eqd_sqnorm_partials: with 0 the norm would read as 0 and clipping would silently not run
  if (!w || !g || !m || !v || !sq_partial || n < 0 || step < 1 || n_partial <= 0 || n_partial > 1024)
    return EQD_ERR_BAD_ARG;
  if (n == 0) return EQD_OK;
  const float bc1 = 1.f - powf(beta1, (float)step), bc2 = 1.f - powf(beta2, (float)step);
  eqd::clip_adam_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      w, g, m, v, n, sq_partial, n_partial, max_norm, lr, beta1, beta2, eps, weight_decay, bc1, bc2, scale_extra, norm_out);
  EQD_CUDA_LAUNCH_CHECK();
  return EQD_OK;
}
