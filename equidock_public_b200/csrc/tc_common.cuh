// wgmma / TMA / mbarrier primitives shared by the tensor-core kernels (sm_90a inline PTX).
//
// Numerics: every GEMM runs as "bf16x6": both operands are split into three bf16 terms
// (v ~ v0 + v1 + v2, round-to-nearest at each level, 24 mantissa bits in total) and the six products
// a0w0, a0w1, a1w0, a0w2, a1w1, a2w0 are accumulated in fp32 registers, smallest first.
//
// Operand conventions (a tile of 128 rows = two warpgroups x 64 rows; in the epilogues thread r <-> row r):
//   A : shared memory, written by the row's threads as bf16x3 (a_store8), canonical K-major no-swizzle layout
//       of 8x8 "core matrices" (128 contiguous bytes); or registers (RS form): an fp32 accumulator fragment split into
//       bf16x3 A fragments in place (acc_to_a_split3), so a GEMM can consume the previous one's epilogue directly.
//   B : shared memory, same canonical layout; descriptor = start address, LBO (stride between core matrices
//       along K), SBO (along N).
//   D : fp32 accumulator fragments of each warpgroup's 64 rows, stored to a row-major shared-memory tile
//       (wg_store_d) from which every thread reads its own row.
//
// Product count P (template parameter of the GEMM and split helpers, default 6): P = 6 is bf16x6 as above; P = 3 is
// "bf16x3", the opt-in mode of the 64-wide layers (eqd_layer_params.mma_products): only the two leading split terms of
// each operand are used and the three products a1w0, a0w1, a0w0 are accumulated (same order, the product loop starts at
// 3).  Each product then carries a relative error of about 2^-16 instead of 2^-24.  With P = 3 the helpers compute and
// store no third A split; B operands keep their three splits in memory (the third is not read).
#pragma once
#include "common.cuh"

namespace eqd {

__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(unsigned long long* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity) {
  unsigned addr = smem_u32(bar);
  unsigned done = 0;
  while (!done) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done) : "r"(addr), "r"(parity) : "memory");
  }
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// TMA 1-D bulk copy global -> shared, completion signalled on an mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, unsigned bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void cp_async8(void* dst, const void* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(smem_u32(dst)), "l"(src));
}
__device__ __forceinline__ void cp_async4(void* dst, const void* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(dst)), "l"(src));
}
// Generic-proxy shared-memory writes (A operands) made visible to the tensor cores' async proxy; callers follow it
// with the barrier that hands the operand to the warpgroups issuing the MMAs.
__device__ __forceinline__ void tc_fence_before() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// No-swizzle canonical shared-memory matrix descriptor (sm_90 wgmma): lbo / sbo in bytes
__device__ __forceinline__ unsigned long long b_desc_ex(unsigned saddr, unsigned lbo, unsigned sbo) {
  return (unsigned long long)((saddr >> 4) & 0x3FFF) | ((unsigned long long)((lbo >> 4) & 0x3FFF) << 16) |
         ((unsigned long long)((sbo >> 4) & 0x3FFF) << 32);
}

// wgmma.mma_async m64nNk16, D fp32 in registers (+=), A and B bf16 from shared-memory descriptors;
// TB = 1 reads B as MN-major ([K][N]).  scale_d = 0 starts a fresh accumulator.
template <int N, int TB>
struct Wgmma;
template <int TB>
struct Wgmma<16, TB> {
  static __device__ __forceinline__ void mma(float (&d)[8], unsigned long long a, unsigned long long b, int scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, %11;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(a), "l"(b), "r"(scale_d), "n"(TB));
  }
};
template <int TB>
struct Wgmma<64, TB> {
  static __device__ __forceinline__ void mma(float (&d)[32], unsigned long long a, unsigned long long b, int scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, %35;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a), "l"(b), "r"(scale_d), "n"(TB));
  }
};
template <int TB>
struct Wgmma<80, TB> {
  static __device__ __forceinline__ void mma(float (&d)[40], unsigned long long a, unsigned long long b, int scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %42, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n80k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39}, %40, %41, p, 1, 1, 0, %43;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39])
        : "l"(a), "l"(b), "r"(scale_d), "n"(TB));
  }
};

// RS form: A from registers (4 x bf16x2 per thread per k16 block, the m16n8k16 A-fragment layout of the warp's 16 rows),
// B from a shared-memory descriptor.
template <int N, int TB>
struct WgmmaRS;
template <int TB>
struct WgmmaRS<64, TB> {
  static __device__ __forceinline__ void mma(float (&d)[32], const unsigned (&a)[4], unsigned long long b, int scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, %38;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(scale_d), "n"(TB));
  }
};

// bf16x6 GEMM of one 64-row slab on the calling warpgroup: d (+)= sum over the last P of the 6 split products (smallest
// terms first) and k-blocks [0, kblocks) of A[split][kb] . B[split][kb]^T; a_desc(split, kb) / b_desc(split, kb) give
// the operand descriptors.  hi_only: just the leading bf16 x bf16 product.  The _issue form returns with the MMAs in
// flight (one commit group; wg_mma_wait completes them), wg_gemm6 with the MMAs complete.
template <int N, int TB = 0, int P = 6, class AD, class BD>
__device__ __forceinline__ void wg_gemm6_issue(float (&d)[N / 2], AD a_desc, BD b_desc, int kblocks, bool accumulate,
                                               bool hi_only = false) {
  static_assert(P == 6 || P == 3, "bf16x6 or bf16x3");
  const int pa[6] = {2, 0, 1, 1, 0, 0}, pb[6] = {0, 2, 1, 0, 1, 0};
  asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
  int scale_d = accumulate ? 1 : 0;
#pragma unroll
  for (int pr = hi_only ? 5 : 6 - P; pr < 6; ++pr)
    for (int kb = 0; kb < kblocks; ++kb) {
      Wgmma<N, TB>::mma(d, a_desc(pa[pr], kb), b_desc(pb[pr], kb), scale_d);
      scale_d = 1;
    }
  asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
}
// waits until at most PENDING of the warpgroup's MMA groups (the most recently committed) are in flight; the accumulators
// handed in (those of an older group) are not touched before it
template <int PENDING = 0, int M>
__device__ __forceinline__ void wg_mma_wait(float (&d)[M]) {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(PENDING) : "memory");
#pragma unroll
  for (int i = 0; i < M; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
template <int N, int TB = 0, int P = 6, class AD, class BD>
__device__ __forceinline__ void wg_gemm6(float (&d)[N / 2], AD a_desc, BD b_desc, int kblocks, bool accumulate,
                                         bool hi_only = false) {
  wg_gemm6_issue<N, TB, P>(d, a_desc, b_desc, kblocks, accumulate, hi_only);
  asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
}
// wg_gemm6_issue with A from registers: a[split][kb] are the bf16x3 A fragments (acc_to_a_split3), same product order
// (P = 3: a[2] is not read); HI_ONLY: just the leading bf16 x bf16 product.  Returns with the MMAs in flight (wg_mma_wait).
template <int N, int KB, int TB = 0, bool HI_ONLY = false, int P = 6, class BD>
__device__ __forceinline__ void wg_gemm6_rs_issue(float (&d)[N / 2], const unsigned (&a)[3][KB][4], BD b_desc, bool accumulate) {
  static_assert(P == 6 || P == 3, "bf16x6 or bf16x3");
  constexpr int pa[6] = {2, 0, 1, 1, 0, 0}, pb[6] = {0, 2, 1, 0, 1, 0};
  asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
  int scale_d = accumulate ? 1 : 0;
#pragma unroll
  for (int pr = HI_ONLY ? 5 : 6 - P; pr < 6; ++pr)
#pragma unroll
    for (int kb = 0; kb < KB; ++kb) {
      WgmmaRS<N, TB>::mma(d, a[pa[pr]][kb], b_desc(pb[pr], kb), scale_d);
      scale_d = 1;
    }
  asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
}

// A operand of a tile of R rows in shared memory, canonical K-major no-swizzle layout of 8 x 16-byte core matrices:
//   byte offset of (split s, k-block kb, 8-channel half kh, row) = s * split_bytes + kb * 32R + kh * 16R + (row / 8) * 128
//   + (row % 8) * 16.  The descriptor of warpgroup h's 64-row slab starts 1024 h bytes in (LBO = 16R, SBO = 128).
template <int R>
__device__ __forceinline__ unsigned long long a_desc_at(unsigned a_saddr, unsigned split_bytes, int wgi, int s, int kb) {
  return b_desc_ex(a_saddr + s * split_bytes + kb * (32 * R) + wgi * 1024, 16 * R, 128);
}
// 8 consecutive channels [c, c + 8) of `row` (c a multiple of 8), as three packed bf16x3 split rows (P = 3: two)
template <int R, int P = 6>
__device__ __forceinline__ void a_store8(unsigned char* a, unsigned split_bytes, int row, int c, const unsigned* p0,
                                         const unsigned* p1, const unsigned* p2) {
  unsigned char* base = a + (c >> 4) * (32 * R) + ((c >> 3) & 1) * (16 * R) + (row >> 3) * 128 + (row & 7) * 16;
  *reinterpret_cast<uint4*>(base) = make_uint4(p0[0], p0[1], p0[2], p0[3]);
  *reinterpret_cast<uint4*>(base + split_bytes) = make_uint4(p1[0], p1[1], p1[2], p1[3]);
  if constexpr (P == 6) *reinterpret_cast<uint4*>(base + 2 * split_bytes) = make_uint4(p2[0], p2[1], p2[2], p2[3]);
}

// wgmma m64nN accumulator fragment of warpgroup thread t -> rows [0, 64) of a row-major fp32 tile (ld floats per row)
template <int N>
__device__ __forceinline__ void wg_store_d(float* tile, int ld, const float (&d)[N / 2], int t) {
  const int row = (t >> 5) * 16 + ((t & 31) >> 2), col = 2 * (t & 3);
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
    *reinterpret_cast<float2*>(tile + row * ld + 8 * j + col) = make_float2(d[4 * j], d[4 * j + 1]);
    *reinterpret_cast<float2*>(tile + (row + 8) * ld + 8 * j + col) = make_float2(d[4 * j + 2], d[4 * j + 3]);
  }
}

// ---- bf16x3 split of register tiles, A-operand stores, result-tile loads ---------------------------
__device__ __forceinline__ unsigned cvt_bf16x2(float hi, float lo) {
  unsigned d;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(hi), "f"(lo));
  return d;
}
// (v0, v1) -> three packed bf16x2 words (v0 in the low half = even k); P = 3: the first two only (p2 is not written)
template <int P = 6>
__device__ __forceinline__ void split3_pair(float v0, float v1, unsigned& p0, unsigned& p1, unsigned& p2) {
  p0 = cvt_bf16x2(v1, v0);
  // v - hi, exact: hi is v rounded to bf16
  const float r0 = v0 - __uint_as_float(p0 << 16), r1 = v1 - __uint_as_float(p0 & 0xFFFF0000u);
  p1 = cvt_bf16x2(r1, r0);
  if constexpr (P == 6) p2 = cvt_bf16x2(r1 - __uint_as_float(p1 & 0xFFFF0000u), r0 - __uint_as_float(p1 << 16));
}
// 32 fp32 values = channels [c0, c0 + 32) of `row` -> bf16x3 -> A operand
template <int R>
__device__ __forceinline__ void store_half_split3(unsigned char* a, unsigned split_bytes, int row, int c0, const float (&v)[32]) {
  unsigned p0[16], p1[16], p2[16];
#pragma unroll
  for (int c = 0; c < 16; ++c) split3_pair(v[2 * c], v[2 * c + 1], p0[c], p1[c], p2[c]);
#pragma unroll
  for (int j = 0; j < 4; ++j) a_store8<R>(a, split_bytes, row, c0 + 8 * j, p0 + 4 * j, p1 + 4 * j, p2 + 4 * j);
}
// 8 fp32 values + 8 zeros = channels [c0, c0 + 16) (one k-block) of `row` -> bf16x3 -> A operand
template <int R>
__device__ __forceinline__ void store_extra8_split3(unsigned char* a, unsigned split_bytes, int row, int c0, const float (&t)[8]) {
  unsigned p0[8], p1[8], p2[8];
#pragma unroll
  for (int c = 0; c < 4; ++c) split3_pair(t[2 * c], t[2 * c + 1], p0[c], p1[c], p2[c]);
#pragma unroll
  for (int c = 4; c < 8; ++c) p0[c] = p1[c] = p2[c] = 0u;
  a_store8<R>(a, split_bytes, row, c0, p0, p1, p2);
  a_store8<R>(a, split_bytes, row, c0 + 8, p0 + 4, p1 + 4, p2 + 4);
}
// m64nN fp32 accumulator fragment (N = 16 KB columns) -> bf16x3 A fragments of an RS wgmma whose K runs over those
// columns.  The accumulator's (row, column) ownership is the A fragment's (row, k) ownership: d[8kb + 2i], d[8kb + 2i + 1]
// hold (row g + 8 (i & 1), k = 16 kb + 8 (i >> 1) + 2 (lane & 3) + {0, 1}) = A register i of k-block kb.
template <int KB, int P = 6>
__device__ __forceinline__ void acc_to_a_split3(const float (&v)[8 * KB], unsigned (&a)[3][KB][4]) {
#pragma unroll
  for (int kb = 0; kb < KB; ++kb)
#pragma unroll
    for (int i = 0; i < 4; ++i) split3_pair<P>(v[8 * kb + 2 * i], v[8 * kb + 2 * i + 1], a[0][kb][i], a[1][kb][i], a[2][kb][i]);
}
// bf16x3 RS A fragments (k = 64 channels, 4 k-blocks) of warpgroup thread t from 64 fp32 rows of 64 channels staged in
// shared memory by 16-byte chunks, chunk k4 of row r at position k4 ^ stage_swz(r) (the fragment loads are then free of
// bank conflicts).  Same split as acc_to_a_split3 on the same values.
__device__ __forceinline__ int stage_swz(int row) { return (row & 3) << 1; }
// Columns [col0, col0 + 64) of rows row0 .. row0 + 63 of a [n][ld] fp32 array -> that staging layout by cp.async (one
// commit group; rows from nvalid on are zero-filled), issued by the 128 threads t of a warpgroup, 16 lanes per row.
__device__ __forceinline__ void stage_rows64(float* rows, const float* src, int ld, int col0, long row0, int nvalid, int t) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int idx = i * 128 + t, row = idx >> 4, k4 = idx & 15;
    const bool ok = row < nvalid;
    cp_async16(rows + row * 64 + ((k4 ^ stage_swz(row)) << 2), src + (row0 + (ok ? row : 0)) * ld + col0 + 4 * k4, ok);
  }
  cp_async_commit();
}
template <int P = 6>
__device__ __forceinline__ void staged_rows_to_a_split3(const float* rows, int t, unsigned (&a)[3][4][4]) {
  const int g = (t >> 5) * 16 + ((t & 31) >> 2), c = t & 3;
#pragma unroll
  for (int kb = 0; kb < 4; ++kb)
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int row = g + 8 * (i & 1), k4 = 4 * kb + 2 * (i >> 1) + (c >> 1);
      const float2 v = *reinterpret_cast<const float2*>(rows + row * 64 + ((k4 ^ stage_swz(row)) << 2) + 2 * (c & 1));
      split3_pair<P>(v.x, v.y, a[0][kb][i], a[1][kb][i], a[2][kb][i]);
    }
}
// The same staged values unsplit, in the m64n64 accumulator layout (the A fragments' ownership: v[8 kb + 2 i + e] is
// register i, element e of k-block kb): acc_to_a_split3<4> on v gives the fragments of staged_rows_to_a_split3.
__device__ __forceinline__ void staged_rows_to_frag(const float* rows, int t, float (&v)[32]) {
  const int g = (t >> 5) * 16 + ((t & 31) >> 2), c = t & 3;
#pragma unroll
  for (int kb = 0; kb < 4; ++kb)
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int row = g + 8 * (i & 1), k4 = 4 * kb + 2 * (i >> 1) + (c >> 1);
      const float2 x = *reinterpret_cast<const float2*>(rows + row * 64 + ((k4 ^ stage_swz(row)) << 2) + 2 * (c & 1));
      v[8 * kb + 2 * i] = x.x;
      v[8 * kb + 2 * i + 1] = x.y;
    }
}
// Row statistics in the summation order of a row-per-thread epilogue: per 32-column half ch of the row, chain k = 0..3 adds
// the columns 32 ch + 4 c4 + k for c4 = 0..7 in turn.  In the accumulator layout lane c of a quad holds the columns
// 8 j + 2 c + e (e = 0, 1), so chain k = 2 (c & 1) + e alternates between lane c and lane c ^ 2; each lane runs its two
// chains from its own values v and those of lane c ^ 2 (pv), and lane c ^ 1 runs the other two.
// Returns term c4 of chain 2 (lane & 1) + e of fragment row h (row g + 8 h).
__device__ __forceinline__ float chain_val(const float (&v)[32], const float (&pv)[32], int h, int ch, int c4, int e) {
  const int i = 4 * (4 * ch + (c4 >> 1)) + 2 * h + e;
  const bool own = ((c4 & 1) == 0) == ((threadIdx.x & 2) == 0);
  return own ? v[i] : pv[i];
}
// barrier of one warpgroup (128 threads) on named barrier `id`; the _and form also returns whether pred holds on all
__device__ __forceinline__ void wg_barrier(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }
__device__ __forceinline__ bool wg_barrier_and(int id, bool pred) {
  unsigned all;
  asm volatile(
      "{\n\t.reg .pred p, q;\n\tsetp.ne.u32 p, %1, 0;\n\t"
      "bar.red.and.pred q, %2, 128, p;\n\tselp.u32 %0, 1, 0, q;\n\t}"
      : "=r"(all) : "r"((unsigned)pred), "r"(id) : "memory");
  return all != 0;
}
// this thread's 32 channels of its row from a row-major fp32 tile
__device__ __forceinline__ void tile_ld32f(const float* tile, int ld, int row, int c0, float (&v)[32]) {
  const float4* s = reinterpret_cast<const float4*>(tile + row * ld + c0);
#pragma unroll
  for (int c4 = 0; c4 < 8; ++c4) {
    float4 t = s[c4];
    v[c4 * 4] = t.x; v[c4 * 4 + 1] = t.y; v[c4 * 4 + 2] = t.z; v[c4 * 4 + 3] = t.w;
  }
}

}  // namespace eqd
