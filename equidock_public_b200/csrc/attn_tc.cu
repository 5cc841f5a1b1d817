// Segmented cross attention of an IEGMN layer (rigid_docking_model.py:46-64, 247-256) on the tensor cores (wgmma,
// bf16x6):   mu_i = sum_j softmax_j(q_i . k_j) v_j   over the partner protein's nodes j
// (the per-pair block of the reference's dense masked softmax; no 1/sqrt(d)).
//
// K and V of every node arrive as bf16x3 8-node blocks (written by the projection kernel), so a run of 8 blocks (64 keys)
// is TMA-bulk-copied straight into shared memory as a wgmma B operand:
//   S = Q K^T   : A = Q (bf16x3), B = K blocks, K-major  (n = key, k = d)
//   O += P V    : A = P (bf16x3), B = V blocks, MN-major (k = key, n = d)
// Two passes over the keys (row maxima first, then exp / P.V) instead of an online softmax: the extra S GEMMs
// are cheap on the tensor pipe and O never has to be rescaled.
//
// Layer 0 (attention0_tc_kernel): a tile = 128 query nodes of one protein; one CTA of 256 threads (2 threads per query
// row, two 64-row warpgroup slabs in the GEMMs); A operands in shared memory, the P region also holds the fp32 S and O
// tiles between the MMAs and the threads that read them.  The 64-wide layers: attention64_tc_kernel below.
#include "tc_common.cuh"

namespace eqd {

#define AT_THREADS 256
#define AT_KEYS 64            // keys per chunk = 8 blocks
#define AT_CHUNK_BYTES 8192   // per split
#define AT_A_SPLIT 16384      // Q and P operands: 128 rows x 64 bf16 per split
#define AT_LD 68              // fp32 row stride of the S / O tiles

// The 69-wide layer 0: the tensor cores handle channels 0..63 exactly as in a 64-wide layer; channels 64..68 of
// Q, K, V (fp32 in x5[n][16] = [K64..67 | V64..67 | K68 V68 | Q64..68 | 0], written by the layer-0 projection) are a
// rank-5 update of the scores and five extra output columns, done with plain FMAs next to the exp().
struct AtGroupSmem {
  unsigned char k[2][3][AT_CHUNK_BYTES];  // double-buffered K chunks (3 splits)
  unsigned char v[2][3][AT_CHUNK_BYTES];
  float red[EQD_TM * 2];
  float x5c[2][AT_KEYS * 16];   // x5 rows of the K chunk in flight (same double buffering as k)
  float red5[EQD_TM * 2 * 5];
};
struct AtSmem {
  unsigned char qa[3 * AT_A_SPLIT];   // Q (A of S = Q K^T)
  unsigned char pa[3 * AT_A_SPLIT];   // P (A of O = P V), or the fp32 S / O tile [128][AT_LD]
  AtGroupSmem grp;
  unsigned long long k_bar[2], v_bar[2];
};

__global__ void __launch_bounds__(AT_THREADS, 1)
attention0_tc_kernel(eqd_graph g, const float* __restrict__ proj, int pw, const unsigned char* __restrict__ kv,
                    long kv_split_stride, const float* __restrict__ x5, float* __restrict__ mu, int ldmu) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  AtSmem& S = *reinterpret_cast<AtSmem*>(smem_raw);
  const int tid = threadIdx.x, q = tid, half = q >> 7, r = q & 127, wgi = tid >> 7;
  AtGroupSmem& G = S.grp;
  if (tid == 0) {
    for (int b = 0; b < 2; ++b) {
      mbar_init(&S.k_bar[b], 1);
      mbar_init(&S.v_bar[b], 1);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const unsigned k_saddr = smem_u32(G.k), v_saddr = smem_u32(G.v);
  const unsigned qa_saddr = smem_u32(S.qa), pa_saddr = smem_u32(S.pa);
  float* const dtile = reinterpret_cast<float*>(S.pa);
  unsigned kph[2] = {0, 0}, vph[2] = {0, 0};
  const int B = g.n_pairs;
  const unsigned char* k_g = kv;                              // which = 0
  const unsigned char* v_g = kv + 3 * kv_split_stride;        // which = 1

  // a chunk of K or V blocks; x5buf >= 0: also the fp32 x5 rows of those 64 keys (they travel with the K chunks)
  auto load_chunk = [&](const unsigned char* src, unsigned char (*dst)[AT_CHUNK_BYTES], unsigned long long* bar, int blk0,
                        int x5buf) {
    if (q == 0) {
      const bool with5 = x5buf >= 0;
      mbar_expect_tx(bar, 3 * AT_CHUNK_BYTES + (with5 ? AT_KEYS * 64 : 0));
#pragma unroll
      for (int s = 0; s < 3; ++s) bulk_g2s(dst[s], src + s * kv_split_stride + (long)blk0 * 1024, AT_CHUNK_BYTES, bar);
      if (with5) bulk_g2s(G.x5c[x5buf], x5 + (long)blk0 * 8 * 16, AT_KEYS * 64, bar);
    }
  };
  // s[i] += <Q5, K5[key i of my half]>   (keys are uniform across the warp: broadcast shared loads)
  auto add_s5 = [&](float (&s)[32], const float* xc, const float (&q5)[5]) {
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const float* row = xc + (half * 32 + i) * 16;
      const float4 k4 = *reinterpret_cast<const float4*>(row);
      const float k8 = row[8];
      s[i] += q5[0] * k4.x + q5[1] * k4.y + q5[2] * k4.z + q5[3] * k4.w + q5[4] * k8;
    }
  };
  // S = Q K^T for one 64-key chunk in K buffer `kb_` -> the fp32 tile in the P region.  hi_only: just the leading
  // bf16 x bf16 product (4 MMAs instead of 24) -- enough for pass 1, which only needs each row's maximum to within a few
  // units to keep exp() in range; the softmax result does not depend on which shift is subtracted.  The caller makes
  // sure nobody still reads the P region.
  auto gemm_s = [&](int kb_, bool hi_only) {
    float d[32];
    wg_gemm6<64>(d, [&](int sp, int kb) { return a_desc_at<EQD_TM>(qa_saddr, AT_A_SPLIT, wgi, sp, kb); },
                 [&](int sp, int kk) { return b_desc_ex(k_saddr + (kb_ * 3 + sp) * AT_CHUNK_BYTES + kk * 256, 128, 1024); },
                 4, false, hi_only);
    wg_store_d<64>(dtile + wgi * 64 * AT_LD, AT_LD, d, tid & 127);
  };
  // O = P V for one chunk in V buffer `vb_` -> the fp32 tile in the P region (once every MMA has read P)
  auto gemm_pv = [&](int vb_) {
    float d[32];
    wg_gemm6<64, 1>(d, [&](int sp, int kb) { return a_desc_at<EQD_TM>(pa_saddr, AT_A_SPLIT, wgi, sp, kb); },
                    [&](int sp, int kk) { return b_desc_ex(v_saddr + (vb_ * 3 + sp) * AT_CHUNK_BYTES + kk * 2048, 1024, 128); },
                    4, false);
    __syncthreads();
    wg_store_d<64>(dtile + wgi * 64 * AT_LD, AT_LD, d, tid & 127);
  };

  for (int tile = blockIdx.x; tile < g.n_node_tiles; tile += gridDim.x) {
    const int seg = g.node_tiles[2 * tile], node0 = g.node_tiles[2 * tile + 1];
    const int nvalid = min(EQD_TM, g.seg_ptr[seg + 1] - node0);
    const int pseg = seg < B ? seg + B : seg - B;
    const int j0 = g.seg_ptr[pseg], j1 = g.seg_ptr[pseg + 1];
    const int blk_lo = j0 >> 3, blk_hi = (j1 + 7) >> 3;
    const int nchunks = (blk_hi - blk_lo + 7) >> 3;
    const int node = node0 + r;
    const bool valid = r < nvalid;
    if (nchunks > 0) load_chunk(k_g, G.k[0], &S.k_bar[0], blk_lo, 0);
    float q5[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
    if (valid) {
#pragma unroll
      for (int e = 0; e < 5; ++e) q5[e] = x5[(long)node * 16 + 10 + e];
    }
    {  // Q row -> bf16x3 -> A
      float v[32];
      const float4* sp = reinterpret_cast<const float4*>(proj + (long)node * pw + 128 + half * 32);
#pragma unroll
      for (int c4 = 0; c4 < 8; ++c4) {
        float4 t = valid ? sp[c4] : make_float4(0.f, 0.f, 0.f, 0.f);
        v[c4 * 4] = t.x; v[c4 * 4 + 1] = t.y; v[c4 * 4 + 2] = t.z; v[c4 * 4 + 3] = t.w;
      }
      store_half_split3<EQD_TM>(S.qa, AT_A_SPLIT, r, half * 32, v);
    }
    tc_fence_before();
    __syncthreads();
    // ---------------- pass 1: row maxima ----------------------------------------------------------------
    float mx = -INFINITY;
    for (int c = 0; c < nchunks; ++c) {
      const int kb_ = c & 1;
      mbar_wait(&S.k_bar[kb_], kph[kb_]);
      kph[kb_] ^= 1;
      // the other K buffer was last read by the S GEMM of chunk c-1, complete before the last barrier: prefetch into it
      if (c + 1 < nchunks) load_chunk(k_g, G.k[kb_ ^ 1], &S.k_bar[kb_ ^ 1], blk_lo + 8 * (c + 1), kb_ ^ 1);
      else load_chunk(k_g, G.k[kb_ ^ 1], &S.k_bar[kb_ ^ 1], blk_lo, kb_ ^ 1);   // first chunk of pass 2
      gemm_s(kb_, true);
      __syncthreads();
      float s[32];
      tile_ld32f(dtile, AT_LD, r, half * 32, s);
      add_s5(s, G.x5c[kb_], q5);
      const int key0 = (blk_lo + 8 * c) * 8 + half * 32;
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        int kn = key0 + i;
        mx = fmaxf(mx, (kn >= j0 && kn < j1) ? s[i] : -INFINITY);
      }
      __syncthreads();  // S drained before the next S GEMM overwrites it
    }
    G.red[r * 2 + half] = mx;
    __syncthreads();
    mx = fmaxf(G.red[r * 2], G.red[r * 2 + 1]);
    // ---------------- pass 2: P = exp(S - max), O += P V ----------------------------------------------------
    float l = 0.f;
    float o_acc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) o_acc[i] = 0.f;
    if (nchunks > 0) load_chunk(v_g, G.v[0], &S.v_bar[0], blk_lo, -1);
    float o5[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
    for (int c = 0; c < nchunks; ++c) {
      const int kb_ = (nchunks + c) & 1, vb_ = c & 1;   // K buffers keep alternating after pass 1
      mbar_wait(&S.k_bar[kb_], kph[kb_]);
      kph[kb_] ^= 1;
      if (c + 1 < nchunks) {
        load_chunk(k_g, G.k[kb_ ^ 1], &S.k_bar[kb_ ^ 1], blk_lo + 8 * (c + 1), kb_ ^ 1);
        load_chunk(v_g, G.v[vb_ ^ 1], &S.v_bar[vb_ ^ 1], blk_lo + 8 * (c + 1), -1);   // its last reader (P V of c-1) is done
      }
      gemm_s(kb_, false);
      __syncthreads();
      float s[32];
      tile_ld32f(dtile, AT_LD, r, half * 32, s);
      add_s5(s, G.x5c[kb_], q5);
      const int key0 = (blk_lo + 8 * c) * 8 + half * 32;
      float l4[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        int kn = key0 + i;
        float pj = (kn >= j0 && kn < j1) ? expf(s[i] - mx) : 0.f;
        s[i] = pj;
        l4[i & 3] += pj;
        {   // the five extra output columns: o5 += p V5[key]
          const float* row = G.x5c[kb_] + (half * 32 + i) * 16;
          const float4 v4 = *reinterpret_cast<const float4*>(row + 4);
          o5[0] = fmaf(pj, v4.x, o5[0]);
          o5[1] = fmaf(pj, v4.y, o5[1]);
          o5[2] = fmaf(pj, v4.z, o5[2]);
          o5[3] = fmaf(pj, v4.w, o5[3]);
          o5[4] = fmaf(pj, row[9], o5[4]);
        }
      }
      l += (l4[0] + l4[1]) + (l4[2] + l4[3]);
      __syncthreads();  // every S value is in registers: the P splits may overwrite the S tile
      store_half_split3<EQD_TM>(S.pa, AT_A_SPLIT, r, half * 32, s);
      tc_fence_before();
      __syncthreads();
      mbar_wait(&S.v_bar[vb_], vph[vb_]);
      vph[vb_] ^= 1;
      gemm_pv(vb_);
      __syncthreads();
      // The tensor core truncates (round-toward-zero) every time it adds into an fp32 accumulator, a systematic
      // bias that grows with the number of accumulation steps; each 64-key chunk is therefore accumulated on its
      // own (4 full-magnitude steps) and the chunks are summed here with round-to-nearest FADDs.
      {
        float oc[32];
        tile_ld32f(dtile, AT_LD, r, half * 32, oc);
#pragma unroll
        for (int i = 0; i < 32; ++i) o_acc[i] += oc[i];
      }
      // Every thread has read its O row (the next S tile overwrites it), and has observed this chunk's v_bar phase
      // before the V refill two chunks ahead re-arms that mbarrier.
      __syncthreads();
    }
    // ---------------- mu = O / l -----------------------------------------------------------------------------
    G.red[r * 2 + half] = l;
    {
#pragma unroll
      for (int e = 0; e < 5; ++e) G.red5[(r * 2 + half) * 5 + e] = o5[e];
    }
    __syncthreads();
    l = G.red[r * 2] + G.red[r * 2 + 1];
    {
      const float inv = l > 0.f ? 1.f / l : 0.f;
      if (valid && half == 0) {   // mu[64..68], then zeros up to the row stride
        float e8[8];
#pragma unroll
        for (int e = 0; e < 5; ++e) e8[e] = (G.red5[r * 10 + e] + G.red5[r * 10 + 5 + e]) * inv;
        e8[5] = e8[6] = e8[7] = 0.f;
        float4* de = reinterpret_cast<float4*>(mu + (long)node * ldmu + 64);
        de[0] = make_float4(e8[0], e8[1], e8[2], e8[3]);
        de[1] = make_float4(e8[4], e8[5], e8[6], e8[7]);
      }
      if (valid) {
        float4* dst = reinterpret_cast<float4*>(mu + (long)node * ldmu + half * 32);
#pragma unroll
        for (int c4 = 0; c4 < 8; ++c4)
          dst[c4] = make_float4(o_acc[c4 * 4] * inv, o_acc[c4 * 4 + 1] * inv, o_acc[c4 * 4 + 2] * inv, o_acc[c4 * 4 + 3] * inv);
      }
    }
    __syncthreads();
  }
}

// ---- the 64-wide layers ---------------------------------------------------------------------------------------------
// One persistent CTA of two warpgroups per SM.  Each warpgroup runs its own chain of 64-row query tiles (the halves of
// the 128-row node_tiles entries; empty halves are skipped) and synchronises only inside itself: its named barrier, its
// own double-buffered K / V chunks and their mbarriers.  While one chain runs its exp / split epilogue, the other's MMAs
// use the tensor pipe.  Every GEMM is an RS wgmma whose accumulator stays in registers:
//   S = Q K^T : A = Q fragments (bf16x3, built once per tile from the staged Q rows), B = K chunk
//   O = P V   : A = P fragments (exp(S - max) of the S accumulator, split in place), B = V chunk (MN-major)
// The K chunks of both passes and the V chunks form two streams that run one chunk ahead of their use across tile
// boundaries, so the next tile's first K and V chunks land during this tile's last chunk.  The next tile's Q rows are
// cp.async'ed into the staging buffer during this tile.  The chunk walk (8-node blocks from the partner's first block)
// does not depend on the query tile: every per-element sum has the order of the 128-row kernel it replaces.
// P = 3 (bf16x3): pass 2's S and O GEMMs take the three leading products on two-term Q / P splits; pass 1 is hi-only in
// both modes.  The K / V chunks are copied whole (their third split is not read).
#define AT_CHAINS 2

struct __align__(128) AtChainSmem {
  unsigned char k[2][3][AT_CHUNK_BYTES];   // double-buffered K chunks (3 splits)
  unsigned char v[2][3][AT_CHUNK_BYTES];
  float qs[64 * 64];                       // Q rows of the next tile (16-byte chunks swizzled, staged_rows_to_a_split3)
  unsigned long long k_bar[2], v_bar[2];
};

struct AtTile {        // one 64-row query tile
  int node0, nvalid;   // first query node, valid rows (> 0)
  int j0, j1;          // partner key range
  int blk_lo, nchunks; // first 8-node block of the walk, 64-key chunks
};

template <int P>
__global__ void __launch_bounds__(AT_CHAINS * 128, 1)
attention64_tc_kernel(eqd_graph g, const float* __restrict__ proj, const unsigned char* __restrict__ kv,
                      long kv_split_stride, float* __restrict__ mu) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  AtChainSmem& W = reinterpret_cast<AtChainSmem*>(smem_raw)[threadIdx.x >> 7];
  const int tid = threadIdx.x, wgi = tid >> 7, t = tid & 127, lane = t & 31;
  const int bar = 1 + wgi;   // this chain's named barrier
  if (t == 0) {
    for (int b = 0; b < 2; ++b) {
      mbar_init(&W.k_bar[b], 1);
      mbar_init(&W.v_bar[b], 1);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  wg_barrier(bar);
  const unsigned k_saddr = smem_u32(W.k), v_saddr = smem_u32(W.v);
  const int B = g.n_pairs, nht = 2 * g.n_node_tiles, hstride = gridDim.x * AT_CHAINS;
  const unsigned char* k_g = kv;                              // which = 0
  const unsigned char* v_g = kv + 3 * kv_split_stride;        // which = 1

  // The k-th tile of this chain is the half (chain + k hstride) ^ (k & 1): hstride is even, so without the swap a chain
  // would always take the same half of the 128-row tiles, and only second halves can be empty.
  const int chain = blockIdx.x * AT_CHAINS + wgi;
  // the chain's first non-empty tile from its k-th on: returns its k (-1 if none) and its metadata
  auto find_tile = [&](int k, AtTile& m) {
    for (; chain + k * hstride < nht; ++k) {
      const int ht = (chain + k * hstride) ^ (k & 1);
      const int seg = __ldg(g.node_tiles + 2 * (ht >> 1));
      m.node0 = __ldg(g.node_tiles + 2 * (ht >> 1) + 1) + 64 * (ht & 1);
      m.nvalid = min(64, __ldg(g.seg_ptr + seg + 1) - m.node0);
      if (m.nvalid <= 0) continue;
      const int pseg = seg < B ? seg + B : seg - B;
      m.j0 = __ldg(g.seg_ptr + pseg);
      m.j1 = __ldg(g.seg_ptr + pseg + 1);
      m.blk_lo = m.j0 >> 3;
      m.nchunks = (((m.j1 + 7) >> 3) - m.blk_lo + 7) >> 3;
      return k;
    }
    return -1;
  };
  // K (V) chunk stream: the n-th chunk filled / consumed uses buffer n & 1, mbarrier phase (n >> 1) & 1.  A chunk is filled
  // into the buffer that the chunk before it has left, and only after a chain barrier that follows every thread's wait on
  // that chunk: so a K / V mbarrier is re-armed only after all 128 threads of the chain have observed its previous phase.
  unsigned kfill = 0, kcons = 0, vfill = 0, vcons = 0;
  auto fill = [&](unsigned char (*dst)[3][AT_CHUNK_BYTES], unsigned long long* bars, unsigned& n, const unsigned char* src,
                  int blk0) {
    if (t == 0) {
      unsigned long long* b = &bars[n & 1];
      mbar_expect_tx(b, 3 * AT_CHUNK_BYTES);
#pragma unroll
      for (int s = 0; s < 3; ++s) bulk_g2s(dst[n & 1][s], src + s * kv_split_stride + (long)blk0 * 1024, AT_CHUNK_BYTES, b);
    }
    ++n;
  };
  auto consume = [&](unsigned long long* bars, unsigned& n) {
    mbar_wait(&bars[n & 1], (n >> 1) & 1);
    return (int)((n++) & 1);
  };
  auto stage_q = [&](const AtTile& m) { stage_rows64(W.qs, proj, 320, 128, m.node0, m.nvalid, t); };

  // accumulator-fragment rows of this thread: fr0 and fr0 + 8; columns (keys, channels) 8 j + fc + {0, 1}, j = 0..7
  const int fr0 = (t >> 5) * 16 + (lane >> 2), fc = 2 * (lane & 3);
  AtTile cur, nxt;
  int kt = find_tile(0, cur);
  bool k_ahead = false, v_ahead = false;   // the current tile's first K / V chunk is already in flight
  if (kt >= 0) stage_q(cur);
  while (kt >= 0) {
    // The next tile's metadata (dependent global loads) and Q rows are fetched once the first S GEMM of pass 1 is in flight.
    int ktn = -1;
    bool looked = false;
    auto look_ahead = [&]() {
      if (looked) return;
      looked = true;
      ktn = find_tile(kt + 1, nxt);
      if (ktn >= 0) stage_q(nxt);   // the staging buffer is free
    };
    if (cur.nchunks > 0 && !k_ahead) fill(W.k, W.k_bar, kfill, k_g, cur.blk_lo);
    // this tile's Q rows have landed (every thread's own copies, then the barrier for the others')
    cp_async_wait<0>();
    wg_barrier(bar);
    unsigned qf[3][4][4];
    staged_rows_to_a_split3<P>(W.qs, t, qf);
    wg_barrier(bar);   // the staging buffer is free
    auto k_desc = [&](int kb_) {
      return [&, kb_](int sp, int kk) { return b_desc_ex(k_saddr + (kb_ * 3 + sp) * AT_CHUNK_BYTES + kk * 256, 128, 1024); };
    };
    // ---------------- pass 1: row maxima (hi-only S) ----------------------------------------------------------------
    float mx[2] = {-INFINITY, -INFINITY};
    for (int c = 0; c < cur.nchunks; ++c) {
      const int kb_ = consume(W.k_bar, kcons);
      // next in the K stream: chunk c + 1, or the first chunk of pass 2
      fill(W.k, W.k_bar, kfill, k_g, cur.blk_lo + (c + 1 < cur.nchunks ? 8 * (c + 1) : 0));
      float s[32];
      wg_gemm6_rs_issue<64, 4, 0, true>(s, qf, k_desc(kb_), false);
      look_ahead();
      wg_mma_wait(s);
      const int key0 = (cur.blk_lo + 8 * c) * 8 + fc;
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int kn = key0 + 8 * j + e;
          const bool ok = kn >= cur.j0 && kn < cur.j1;
#pragma unroll
          for (int h = 0; h < 2; ++h) mx[h] = fmaxf(mx[h], ok ? s[4 * j + 2 * h + e] : -INFINITY);
        }
      wg_barrier(bar);   // K buffer kb_ read and its phase observed by every thread
    }
    look_ahead();
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
    }
    // ---------------- pass 2: P = exp(S - max), O += P V ------------------------------------------------------------
    float lh[2][2] = {{0.f, 0.f}, {0.f, 0.f}};   // [fragment row][32-key half]: the row-per-thread code's per-half sums
    float o_acc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) o_acc[i] = 0.f;
    if (cur.nchunks > 0 && !v_ahead) fill(W.v, W.v_bar, vfill, v_g, cur.blk_lo);
    for (int c = 0; c < cur.nchunks; ++c) {
      const int kb_ = consume(W.k_bar, kcons);
      const bool last = c + 1 == cur.nchunks;
      if (!last) {
        fill(W.k, W.k_bar, kfill, k_g, cur.blk_lo + 8 * (c + 1));
        fill(W.v, W.v_bar, vfill, v_g, cur.blk_lo + 8 * (c + 1));
      } else if (ktn >= 0 && nxt.nchunks > 0) {   // the next tile's first chunks
        fill(W.k, W.k_bar, kfill, k_g, nxt.blk_lo);
        fill(W.v, W.v_bar, vfill, v_g, nxt.blk_lo);
      }
      float s[32];
      wg_gemm6_rs_issue<64, 4, 0, false, P>(s, qf, k_desc(kb_), false);
      wg_mma_wait(s);
      const int key0 = (cur.blk_lo + 8 * c) * 8 + fc;
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int kn = key0 + 8 * j + e;
          const bool ok = kn >= cur.j0 && kn < cur.j1;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float& x = s[4 * j + 2 * h + e];
            x = ok ? expf(x - mx[h]) : 0.f;
          }
        }
      {  // l: four chains per 32-key half, (l0 + l1) + (l2 + l3), added to the half's running sum
        float ps[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) ps[i] = __shfl_xor_sync(0xffffffffu, s[i], 2);
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int ch = 0; ch < 2; ++ch) {
            float s0 = 0.f, s1 = 0.f;
#pragma unroll
            for (int c4 = 0; c4 < 8; ++c4) {
              s0 = __fadd_rn(s0, chain_val(s, ps, h, ch, c4, 0));
              s1 = __fadd_rn(s1, chain_val(s, ps, h, ch, c4, 1));
            }
            const float sp = __fadd_rn(s0, s1);
            lh[h][ch] = __fadd_rn(lh[h][ch], __fadd_rn(sp, __shfl_xor_sync(0xffffffffu, sp, 1)));
          }
      }
      unsigned pf[3][4][4];
      acc_to_a_split3<4, P>(s, pf);
      const int vb_ = consume(W.v_bar, vcons);
      float o[32];
      wg_gemm6_rs_issue<64, 4, 1, false, P>(o, pf, [&](int sp, int kk) {
        return b_desc_ex(v_saddr + (vb_ * 3 + sp) * AT_CHUNK_BYTES + kk * 2048, 1024, 128); }, false);
      wg_mma_wait(o);
      // The tensor core truncates (round-toward-zero) every time it adds into an fp32 accumulator, a systematic bias that
      // grows with the number of accumulation steps; each 64-key chunk is therefore accumulated on its own (4
      // full-magnitude steps) and the chunks are summed here with round-to-nearest FADDs.
#pragma unroll
      for (int i = 0; i < 32; ++i) o_acc[i] = __fadd_rn(o_acc[i], o[i]);
      wg_barrier(bar);   // K buffer kb_ and V buffer vb_ read and their phases observed by every thread
    }
    k_ahead = v_ahead = ktn >= 0 && nxt.nchunks > 0 && cur.nchunks > 0;
    // ---------------- mu = O / l --------------------------------------------------------------------------------------
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float l = __fadd_rn(lh[h][0], lh[h][1]);
      const float inv = l > 0.f ? 1.f / l : 0.f;
      const int row = fr0 + 8 * h;
      if (row < cur.nvalid) {
        float* dst = mu + (long)(cur.node0 + row) * EQD_HID + fc;
#pragma unroll
        for (int j = 0; j < 8; ++j)
          *reinterpret_cast<float2*>(dst + 8 * j) = make_float2(o_acc[4 * j + 2 * h] * inv, o_acc[4 * j + 2 * h + 1] * inv);
      }
    }
    kt = ktn;
    cur = nxt;
  }
  cp_async_wait<0>();
}

// ---- the 64-wide layers, partner K / V resident in shared memory ------------------------------------------------------
// For batches whose partner proteins all fit (eqd_graph.max_segment_nodes <= AT_RES_MAX_NODES): the unit of work is one
// query protein.  Its partner's K / V chunks (the same 8-block chunks from the partner's first block that
// attention64_tc_kernel streams for every 64-row query tile) are copied once into six resident planes, K and V x 3
// splits, and every query tile of the protein reads them from there: the per-tile chunk stream, its mbarrier waits and
// the chain barriers that protected its refills are gone.  The GEMMs, masks and sums are those of attention64_tc_kernel
// on the same B bytes, so mu is bitwise the same.
//   K split 0 (all that pass 1's hi-only S GEMMs read) lands first under res_k0; the other five planes follow per chunk,
//   chunk c under res_kv[c].  Both chains take the protein's non-empty 64-row halves (chain c: halves c, c + 2, ...); the
//   planes are refilled for the CTA's next protein after a CTA barrier that follows both chains' last tile, so each
//   mbarrier is re-armed only after every thread has observed its previous phase.
#define AT_RES_CHUNKS 4
#define AT_RES_BLOCKS (AT_RES_CHUNKS * 8)
#define AT_RES_PLANE (AT_RES_CHUNKS * AT_CHUNK_BYTES)
// largest partner whose chunk walk fits: a segment that starts mid-block spans ceil(n / 8) + 1 blocks
#define AT_RES_MAX_NODES (8 * (AT_RES_BLOCKS - 1))

struct __align__(128) AtResSmem {
  unsigned char k[3][AT_RES_PLANE];   // resident K chunks, one plane per split
  unsigned char v[3][AT_RES_PLANE];
  float qs[AT_CHAINS][64 * 64];       // per chain: Q rows of its next tile
  unsigned long long res_k0, res_kv[AT_RES_CHUNKS];
};
static_assert(sizeof(AtResSmem) <= 227 * 1024, "resident K / V planes + Q staging exceed the 227 KB of shared memory per CTA");

template <int P>
__global__ void __launch_bounds__(AT_CHAINS * 128, 1)
attention64_res_kernel(eqd_graph g, const float* __restrict__ proj, const unsigned char* __restrict__ kv,
                       long kv_split_stride, float* __restrict__ mu) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  AtResSmem& R = *reinterpret_cast<AtResSmem*>(smem_raw);
  const int tid = threadIdx.x, wgi = tid >> 7, t = tid & 127, lane = t & 31;
  const int bar = 1 + wgi;   // this chain's named barrier
  float* const qs = R.qs[wgi];
  if (tid == 0) {
    mbar_init(&R.res_k0, 1);
    for (int c = 0; c < AT_RES_CHUNKS; ++c) mbar_init(&R.res_kv[c], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const unsigned k_saddr = smem_u32(R.k), v_saddr = smem_u32(R.v);
  const int B = g.n_pairs, nseg = 2 * B;
  const unsigned char* k_g = kv;                              // which = 0
  const unsigned char* v_g = kv + 3 * kv_split_stride;        // which = 1

  // The chain's tiles in order: (segment, half), segments blockIdx.x + i gridDim.x, halves wgi, wgi + 2, ... of each.
  // next_tile: the first one from (seg, h) on; seg = -1 if none.
  auto next_tile = [&](int& seg, int& h) {
    for (; seg < nseg; seg += gridDim.x, h = wgi)
      if (64 * h < __ldg(g.seg_ptr + seg + 1) - __ldg(g.seg_ptr + seg)) return;
    seg = -1;
  };
  auto stage_q = [&](int seg, int h) {
    const int node0 = __ldg(g.seg_ptr + seg) + 64 * h;
    stage_rows64(qs, proj, 320, 128, node0, min(64, __ldg(g.seg_ptr + seg + 1) - node0), t);
  };
  int qseg = blockIdx.x, qh = wgi;   // the chain's next tile to stage
  next_tile(qseg, qh);
  if (qseg >= 0) stage_q(qseg, qh);

  const int fr0 = (t >> 5) * 16 + (lane >> 2), fc = 2 * (lane & 3);
  unsigned phase = 0;   // of every resident-plane mbarrier: one completed phase per loaded segment
  for (int seg = blockIdx.x; seg < nseg; seg += gridDim.x) {
    const int i0 = __ldg(g.seg_ptr + seg), i1 = __ldg(g.seg_ptr + seg + 1);
    if (i1 <= i0) continue;
    const int pseg = seg < B ? seg + B : seg - B;
    const int j0 = __ldg(g.seg_ptr + pseg), j1 = __ldg(g.seg_ptr + pseg + 1);
    const int blk_lo = j0 >> 3, nchunks = (((j1 + 7) >> 3) - blk_lo + 7) >> 3;
    const bool fits = nchunks <= AT_RES_CHUNKS;
    if (tid == 0 && fits) {
      // every mbarrier completes one phase per segment: chunks the partner does not have are plain arrivals
      mbar_expect_tx(&R.res_k0, nchunks * AT_CHUNK_BYTES);
      if (nchunks > 0) bulk_g2s(R.k[0], k_g + (long)blk_lo * 1024, nchunks * AT_CHUNK_BYTES, &R.res_k0);
      for (int c = 0; c < AT_RES_CHUNKS; ++c) {
        unsigned long long* b = &R.res_kv[c];
        if (c >= nchunks) {
          mbar_expect_tx(b, 0);
          continue;
        }
        mbar_expect_tx(b, 5 * AT_CHUNK_BYTES);
        const long off = (long)(blk_lo + 8 * c) * 1024;
#pragma unroll
        for (int s = 0; s < 3; ++s) {
          if (s > 0) bulk_g2s(R.k[s] + c * AT_CHUNK_BYTES, k_g + s * kv_split_stride + off, AT_CHUNK_BYTES, b);
          bulk_g2s(R.v[s] + c * AT_CHUNK_BYTES, v_g + s * kv_split_stride + off, AT_CHUNK_BYTES, b);
        }
      }
    }
    for (int h = wgi; 64 * h < i1 - i0; h += 2) {
      const int node0 = i0 + 64 * h, nvalid = min(64, i1 - node0);
      // this tile's Q rows have landed (every thread's own copies, then the barrier for the others')
      cp_async_wait<0>();
      wg_barrier(bar);
      unsigned qf[3][4][4];
      staged_rows_to_a_split3<P>(qs, t, qf);
      wg_barrier(bar);   // the staging buffer is free: the chain's next tile
      qh += 2;
      next_tile(qseg, qh);
      if (qseg >= 0) stage_q(qseg, qh);
      if (!fits) {   // only reachable if max_segment_nodes understated the batch: no overrun, and NaN marks the rows
        for (int i = t; i < nvalid * EQD_HID; i += 128) mu[(long)node0 * EQD_HID + i] = __int_as_float(0x7fc00000);
        continue;
      }
      auto k_desc = [&](int c) {
        return [&, c](int sp, int kk) { return b_desc_ex(k_saddr + sp * AT_RES_PLANE + c * AT_CHUNK_BYTES + kk * 256, 128, 1024); };
      };
      // ---------------- pass 1: row maxima (hi-only S) --------------------------------------------------------------
      float mx[2] = {-INFINITY, -INFINITY};
      if (nchunks > 0) mbar_wait(&R.res_k0, phase);
      for (int c = 0; c < nchunks; ++c) {
        float s[32];
        wg_gemm6_rs_issue<64, 4, 0, true>(s, qf, k_desc(c), false);
        wg_mma_wait(s);
        const int key0 = (blk_lo + 8 * c) * 8 + fc;
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int kn = key0 + 8 * j + e;
            const bool ok = kn >= j0 && kn < j1;
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) mx[hh] = fmaxf(mx[hh], ok ? s[4 * j + 2 * hh + e] : -INFINITY);
          }
      }
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 1));
        mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 2));
      }
      // ---------------- pass 2: P = exp(S - max), O += P V ----------------------------------------------------------
      float lh[2][2] = {{0.f, 0.f}, {0.f, 0.f}};   // [fragment row][32-key half]: the row-per-thread code's per-half sums
      float o_acc[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) o_acc[i] = 0.f;
      for (int c = 0; c < nchunks; ++c) {
        mbar_wait(&R.res_kv[c], phase);
        float s[32];
        wg_gemm6_rs_issue<64, 4, 0, false, P>(s, qf, k_desc(c), false);
        wg_mma_wait(s);
        const int key0 = (blk_lo + 8 * c) * 8 + fc;
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int kn = key0 + 8 * j + e;
            const bool ok = kn >= j0 && kn < j1;
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
              float& x = s[4 * j + 2 * hh + e];
              x = ok ? expf(x - mx[hh]) : 0.f;
            }
          }
        {  // l: four chains per 32-key half, (l0 + l1) + (l2 + l3), added to the half's running sum
          float ps[32];
#pragma unroll
          for (int i = 0; i < 32; ++i) ps[i] = __shfl_xor_sync(0xffffffffu, s[i], 2);
#pragma unroll
          for (int hh = 0; hh < 2; ++hh)
#pragma unroll
            for (int ch = 0; ch < 2; ++ch) {
              float s0 = 0.f, s1 = 0.f;
#pragma unroll
              for (int c4 = 0; c4 < 8; ++c4) {
                s0 = __fadd_rn(s0, chain_val(s, ps, hh, ch, c4, 0));
                s1 = __fadd_rn(s1, chain_val(s, ps, hh, ch, c4, 1));
              }
              const float sp = __fadd_rn(s0, s1);
              lh[hh][ch] = __fadd_rn(lh[hh][ch], __fadd_rn(sp, __shfl_xor_sync(0xffffffffu, sp, 1)));
            }
        }
        unsigned pf[3][4][4];
        acc_to_a_split3<4, P>(s, pf);
        float o[32];
        wg_gemm6_rs_issue<64, 4, 1, false, P>(o, pf, [&](int sp, int kk) {
          return b_desc_ex(v_saddr + sp * AT_RES_PLANE + c * AT_CHUNK_BYTES + kk * 2048, 1024, 128); }, false);
        wg_mma_wait(o);
        // chunks summed with round-to-nearest FADDs, as in attention64_tc_kernel
#pragma unroll
        for (int i = 0; i < 32; ++i) o_acc[i] = __fadd_rn(o_acc[i], o[i]);
      }
      // ---------------- mu = O / l ------------------------------------------------------------------------------------
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const float l = __fadd_rn(lh[hh][0], lh[hh][1]);
        const float inv = l > 0.f ? 1.f / l : 0.f;
        const int row = fr0 + 8 * hh;
        if (row < nvalid) {
          float* dst = mu + (long)(node0 + row) * EQD_HID + fc;
#pragma unroll
          for (int j = 0; j < 8; ++j)
            *reinterpret_cast<float2*>(dst + 8 * j) = make_float2(o_acc[4 * j + 2 * hh] * inv, o_acc[4 * j + 2 * hh + 1] * inv);
        }
      }
    }
    // both chains' MMAs on the planes are complete and every thread has observed this segment's phases: refill
    __syncthreads();
    if (fits) phase ^= 1;
  }
  cp_async_wait<0>();
}

template <int P>
static int launch_attention64_tc(const eqd_graph* g, const float* proj, const void* kv, float* mu, void* stream) {
  const long split_stride = (long)((g->n_nodes + 7) / 8 + 8) * 1024;
  if (g->max_segment_nodes > 0 && g->max_segment_nodes <= AT_RES_MAX_NODES) {
    const size_t smem = sizeof(AtResSmem);
    EQD_SET_SMEM(attention64_res_kernel<P>, smem);
    const int grid = 2 * g->n_pairs < EQD_SMS ? 2 * g->n_pairs : EQD_SMS;
    attention64_res_kernel<P><<<grid, AT_CHAINS * 128, smem, (cudaStream_t)stream>>>(
        *g, proj, reinterpret_cast<const unsigned char*>(kv), split_stride, mu);
    EQD_CUDA_LAUNCH_CHECK();
    return EQD_OK;
  }
  const size_t smem = AT_CHAINS * sizeof(AtChainSmem);
  EQD_SET_SMEM(attention64_tc_kernel<P>, smem);
  const int nht = 2 * g->n_node_tiles;
  int grid = (nht + AT_CHAINS - 1) / AT_CHAINS;
  if (grid > EQD_SMS) grid = EQD_SMS;
  attention64_tc_kernel<P><<<grid, AT_CHAINS * 128, smem, (cudaStream_t)stream>>>(
      *g, proj, reinterpret_cast<const unsigned char*>(kv), split_stride, mu);
  EQD_CUDA_LAUNCH_CHECK();
  return EQD_OK;
}

}  // namespace eqd

// eqd_attention_tc with the product count of a layer's tensor-core GEMMs (6 or 3, eqd_mma_products); the node stage's
// entry point, not part of the C ABI
int eqd_attention_tc_products(const eqd_graph* g, const float* proj, const void* kv, float* mu, int products, void* stream) {
  if (!g || !proj || !kv || !mu) return EQD_ERR_BAD_ARG;
  if (reinterpret_cast<uintptr_t>(kv) & 15) return EQD_ERR_BAD_ARG;
  if (products != 6 && products != 3) return EQD_ERR_UNSUPPORTED;
  if (g->n_node_tiles <= 0) return EQD_OK;
  return products == 3 ? eqd::launch_attention64_tc<3>(g, proj, kv, mu, stream)
                       : eqd::launch_attention64_tc<6>(g, proj, kv, mu, stream);
}

extern "C" int eqd_attention_tc(const eqd_graph* g, const float* proj, const void* kv, float* mu, void* stream) {
  return eqd_attention_tc_products(g, proj, kv, mu, 6, stream);
}

extern "C" int eqd_attention_tc0(const eqd_graph* g, const float* proj, const void* kv, const float* x5, float* mu,
                                 void* stream) {
  if (!g || !proj || !kv || !x5 || !mu) return EQD_ERR_BAD_ARG;
  if ((reinterpret_cast<uintptr_t>(kv) | reinterpret_cast<uintptr_t>(x5)) & 15) return EQD_ERR_BAD_ARG;
  if (g->n_node_tiles <= 0) return EQD_OK;
  const size_t smem = sizeof(eqd::AtSmem) + 128;
  EQD_SET_SMEM(eqd::attention0_tc_kernel, smem);
  const int grid = g->n_node_tiles < EQD_SMS ? g->n_node_tiles : EQD_SMS;
  const long split_stride = (long)((g->n_nodes + 7) / 8 + 8) * 1024;
  eqd::attention0_tc_kernel<<<grid, AT_THREADS, smem, (cudaStream_t)stream>>>(
      *g, proj, 128 + 3 * 72, reinterpret_cast<const unsigned char*>(kv), split_stride, x5, mu, EQD_H0_PAD);
  EQD_CUDA_LAUNCH_CHECK();
  return EQD_OK;
}
