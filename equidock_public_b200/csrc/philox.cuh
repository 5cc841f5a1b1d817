// Counter-based random numbers shared by the kernels: Philox4x32-10 (Salmon et al., SC'11) and the training-mode dropout
// masks built on it (eqd_dropout, include/eqd_iegmn.h).  Restated in numpy in tests/dropout_masks.py.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/eqd_iegmn.h"

namespace eqd {

// Philox4x32-10: counter c, key k.
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
    k.x += 0x9E3779B9u;
    k.y += 0xBB67AE85u;
  }
  return c;
}

// The four mask words of columns 4*col4 .. 4*col4+3 of one row of a dropout site.
__device__ __forceinline__ uint4 dropout_words(const eqd_dropout& d, int site, int row, int col4) {
  return philox4x32_10(make_uint4((uint32_t)row, (uint32_t)col4, ((uint32_t)d.layer << 2) | (uint32_t)site, (uint32_t)d.rank),
                       make_uint2((uint32_t)d.seed, (uint32_t)(d.seed >> 32)));
}

__device__ __forceinline__ float dropout_apply(float z, uint32_t w, const eqd_dropout& d) {
  return w >= d.threshold ? z * d.scale : 0.f;
}

// Dropout on this thread's rows of a 128-row NN micro-tile (common.cuh: rows row0 + i, columns tx*4 + (j&3) + 32*(j>>2);
// with EXTRA also column 64 + tx in accx).  row0 = the global edge / node id of the thread's first row.
template <bool EXTRA>
__device__ __forceinline__ void dropout_tile(float (&acc)[8][8], float (&accx)[8], const eqd_dropout& d, int site, int row0,
                                             int tx) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const uint4 a = dropout_words(d, site, row0 + i, tx), b = dropout_words(d, site, row0 + i, 8 + tx);
    acc[i][0] = dropout_apply(acc[i][0], a.x, d); acc[i][1] = dropout_apply(acc[i][1], a.y, d);
    acc[i][2] = dropout_apply(acc[i][2], a.z, d); acc[i][3] = dropout_apply(acc[i][3], a.w, d);
    acc[i][4] = dropout_apply(acc[i][4], b.x, d); acc[i][5] = dropout_apply(acc[i][5], b.y, d);
    acc[i][6] = dropout_apply(acc[i][6], b.z, d); acc[i][7] = dropout_apply(acc[i][7], b.w, d);
    if (EXTRA) {
      const uint4 x = dropout_words(d, site, row0 + i, 16 + (tx >> 2));
      const uint32_t wx = (tx & 3) == 0 ? x.x : (tx & 3) == 1 ? x.y : (tx & 3) == 2 ? x.z : x.w;
      accx[i] = dropout_apply(accx[i], wx, d);
    }
  }
}

}  // namespace eqd
