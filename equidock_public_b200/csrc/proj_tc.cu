// Node projections of a layer on the tensor cores (wgmma, bf16x6; att_mlp_Q/K/V :130-140 and the [h_src|h_dst]
// columns of edge_mlp.0 :120, applied per node):
//   proj[n] = [Psrc | Pdst | Q | K | V] = act(h[n] . Wp + b)      (groups of 64 columns, see eqd_layer_params)
// plus, for the tensor-core attention of the same layer, K and V of every node as bf16x3 in 8-node blocks
//   kv[which][split][n/8][d/8][n%8][d%8]   (1 KB per 8 nodes; a run of blocks is a ready wgmma B operand).
// Weight-stationary: the bf16x3 panels (120 KB; 158 KB for the K = 80 layer 0) sit in shared memory for the life of
// the CTA next to the tile's A operand and its fp32 result tile; 2 threads per node row, one 64-row warpgroup slab per
// 128 threads (layer 0 takes 64-row tiles: its larger panels leave room for no more).  eqd_project_tc (the 64-wide
// layers) runs project64_tc_kernel below.
#include "tc_common.cuh"

namespace eqd {

#define PJ_LD 68   // fp32 row stride of the result tile

// Two instances: the 64-wide layers (K = 64, 5 groups) and the 69-wide layer 0 (h = h0, K = 69 padded to 80 = 5 k-blocks;
// the first 64 channels of Q / K / V go where the 64-wide layers put theirs, channels 64..68 of all three form a sixth
// N = 16 group written to x5[n][16] = [K64..67 | V64..67 | K68 V68 | Q64..68 | 0], the layout the layer-0 attention reads).
template <bool L0>
struct PjCfg {
  static constexpr int R = L0 ? 64 : 128;                 // rows per tile
  static constexpr int THREADS = 2 * R;
  static constexpr int KB = L0 ? 5 : 4;                   // k-blocks of 16
  static constexpr int GROUP_BYTES = 64 * KB * 16 * 2 * 3;  // one N = 64 group: 3 splits
  static constexpr int SPLIT_BYTES = 64 * KB * 16 * 2;
  static constexpr int X_SPLIT_BYTES = 16 * KB * 16 * 2;
  static constexpr int W_BYTES = 5 * GROUP_BYTES + (L0 ? 3 * X_SPLIT_BYTES : 0);
  static constexpr int A_SPLIT_BYTES = R * KB * 32;
  static constexpr int NGROUPS = L0 ? 6 : 5;
};

struct PjConsts { float b[336]; };

template <bool L0>
struct PjSmem {
  unsigned char w[PjCfg<L0>::W_BYTES];
  unsigned char a[3 * PjCfg<L0>::A_SPLIT_BYTES];
  float d[PjCfg<L0>::R * PJ_LD];
  unsigned long long w_bar;
};

// bf16x3 block-layout store of 32 consecutive channels [half*32, +32) of node `node`
__device__ __forceinline__ void store_kv_blocks(unsigned char* __restrict__ kv, long split_stride, int node, int half,
                                                const float (&v)[32]) {
  unsigned p0[16], p1[16], p2[16];
#pragma unroll
  for (int c = 0; c < 16; ++c) split3_pair(v[2 * c], v[2 * c + 1], p0[c], p1[c], p2[c]);
  unsigned char* base = kv + (long)(node >> 3) * 1024 + (node & 7) * 16 + half * 512;
#pragma unroll
  for (int j = 0; j < 4; ++j) {  // 4 groups of 8 channels = 16 bytes each
    *reinterpret_cast<uint4*>(base + j * 128) = make_uint4(p0[4 * j], p0[4 * j + 1], p0[4 * j + 2], p0[4 * j + 3]);
    *reinterpret_cast<uint4*>(base + split_stride + j * 128) = make_uint4(p1[4 * j], p1[4 * j + 1], p1[4 * j + 2], p1[4 * j + 3]);
    *reinterpret_cast<uint4*>(base + 2 * split_stride + j * 128) = make_uint4(p2[4 * j], p2[4 * j + 1], p2[4 * j + 2], p2[4 * j + 3]);
  }
}

template <bool L0>
__global__ void __launch_bounds__(PjCfg<L0>::THREADS, 1)
project_tc_kernel(int n_nodes, eqd_layer_params p, const __grid_constant__ PjConsts cst, const float* __restrict__ h, int ldh,
                  float* __restrict__ proj, int pw, unsigned char* __restrict__ kv, long kv_split_stride, float* __restrict__ x5) {
  using C = PjCfg<L0>;
  constexpr int R = C::R;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  PjSmem<L0>& S = *reinterpret_cast<PjSmem<L0>*>(smem_raw);
  const int tid = threadIdx.x, half = tid / R, r = tid % R, warp = tid >> 5, wgi = tid >> 7;
  const int ntiles = (n_nodes + R - 1) / R;
  if (tid == 0) {
    mbar_init(&S.w_bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    mbar_expect_tx(&S.w_bar, C::W_BYTES);
    bulk_g2s(S.w, p.w_proj_tc, C::W_BYTES, &S.w_bar);
  }
  __syncthreads();
  const unsigned w_saddr = smem_u32(S.w), a_saddr = smem_u32(S.a);
  auto a_desc = [&](int s, int kb) { return a_desc_at<R>(a_saddr, C::A_SPLIT_BYTES, wgi, s, kb); };
  float* dslab = S.d + wgi * 64 * PJ_LD;   // this warpgroup's 64 result rows
  mbar_wait(&S.w_bar, 0);
  const float slope = p.leaky_slope;
  const int lane = tid & 31, wrow0 = (warp * 32) % R;   // the warp's 32 rows (of its column half)

  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int node0 = tile * R;
    const int node = node0 + r;
    const bool valid = node < n_nodes;
    {
      float v[32];
      const float4* hp = reinterpret_cast<const float4*>(h + (long)node * ldh + half * 32);
#pragma unroll
      for (int c4 = 0; c4 < 8; ++c4) {
        float4 t = valid ? hp[c4] : make_float4(0.f, 0.f, 0.f, 0.f);
        v[c4 * 4] = t.x; v[c4 * 4 + 1] = t.y; v[c4 * 4 + 2] = t.z; v[c4 * 4 + 3] = t.w;
      }
      if (L0 && half == 0) {   // the 69 - 64 extra channels (h0 is zero-padded to 72) as a fifth k-block
        const float4* ep = reinterpret_cast<const float4*>(h + (long)node * ldh + 64);
        float4 a = valid ? ep[0] : make_float4(0.f, 0.f, 0.f, 0.f), b = valid ? ep[1] : make_float4(0.f, 0.f, 0.f, 0.f);
        float t[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
        store_extra8_split3<R>(S.a, C::A_SPLIT_BYTES, r, 64, t);
      }
      store_half_split3<R>(S.a, C::A_SPLIT_BYTES, r, half * 32, v);
    }
    tc_fence_before();
    __syncthreads();
#pragma unroll 1
    for (int grp = 0; grp < C::NGROUPS; ++grp) {
      if (L0 && grp == 5) {   // channels 64..68 of K, V, Q -> x5 (half-0 threads own the 16 columns)
        float d[8];
        wg_gemm6<16>(d, a_desc, [&](int s, int kb) {
          return b_desc_ex(w_saddr + 5 * C::GROUP_BYTES + s * C::X_SPLIT_BYTES + kb * 512, 256, 128); }, C::KB, false);
        wg_store_d<16>(dslab, PJ_LD, d, tid & 127);
        __syncthreads();
        if (half == 0 && valid) {
          float e[16];
#pragma unroll
          for (int c = 0; c < 16; ++c) {
            const bool act = (c < 4) || c == 8 || (c >= 10 && c < 15);   // K and Q carry the LeakyReLU, V does not
            const float x = S.d[r * PJ_LD + c];
            e[c] = act ? lrelu(x, slope) : x;
          }
          float4* o = reinterpret_cast<float4*>(x5 + (long)node * 16);
#pragma unroll
          for (int c4 = 0; c4 < 4; ++c4) o[c4] = make_float4(e[c4 * 4], e[c4 * 4 + 1], e[c4 * 4 + 2], e[c4 * 4 + 3]);
        }
        continue;
      }
      {
        float d[32];
        wg_gemm6<64>(d, a_desc, [&](int s, int kb) {
          return b_desc_ex(w_saddr + grp * C::GROUP_BYTES + s * C::SPLIT_BYTES + kb * 2048, 1024, 128); }, C::KB, false);
        wg_store_d<64>(dslab, PJ_LD, d, tid & 127);
      }
      __syncthreads();
      float v[32];
      tile_ld32f(S.d, PJ_LD, r, half * 32, v);
      const bool act = (grp == 2 || grp == 3);        // Q, K carry the LeakyReLU
#pragma unroll
      for (int c = 0; c < 32; ++c) {
        float t = v[c] + cst.b[grp * 64 + half * 32 + c];
        v[c] = act ? lrelu(t, slope) : t;
      }
      if (grp < 3 || kv == nullptr) {   // with K/V blocks requested nobody reads the fp32 K / V columns: skip 2 x 256 B / node
        if (L0) {
          if (valid) {
            float4* o = reinterpret_cast<float4*>(proj + (long)node * pw + grp * 64 + half * 32);
#pragma unroll
            for (int c4 = 0; c4 < 8; ++c4) o[c4] = make_float4(v[c4 * 4], v[c4 * 4 + 1], v[c4 * 4 + 2], v[c4 * 4 + 3]);
          }
        } else {
          // back through my row of the result tile so that 8 lanes write one contiguous 128-byte half row (full sectors)
          float* sc = S.d + r * PJ_LD + half * 32;
#pragma unroll
          for (int c4 = 0; c4 < 8; ++c4)
            *reinterpret_cast<float4*>(sc + c4 * 4) = make_float4(v[c4 * 4], v[c4 * 4 + 1], v[c4 * 4 + 2], v[c4 * 4 + 3]);
          __syncwarp();
          float* o = proj + (long)(node0 + wrow0) * pw + grp * 64 + half * 32 + (lane & 7) * 4;
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const int row = i * 4 + (lane >> 3);
            float4 t = *reinterpret_cast<const float4*>(S.d + (wrow0 + row) * PJ_LD + half * 32 + (lane & 7) * 4);
            if (node0 + wrow0 + row < n_nodes) *reinterpret_cast<float4*>(o + (long)row * pw) = t;
          }
        }
      }
      if (valid && grp >= 3 && kv != nullptr)
        store_kv_blocks(kv + (long)(grp - 3) * 3 * kv_split_stride, kv_split_stride, node, half, v);
      __syncthreads();   // the result tile is free for the next group
    }
    __syncthreads();     // A may be overwritten by the next tile
  }
}

// ---- the 64-wide layers ---------------------------------------------------------------------------------------------
// One persistent CTA of two warpgroups per SM sharing the resident 120 KB panels.  Each warpgroup runs its own chain of
// 64-row tiles and synchronises only inside itself (its named barrier).  Per tile: the h rows, cp.async'ed into the
// chain's staging buffer during the previous tile, become bf16x3 RS A fragments once; the five N = 64 groups run as RS
// wgmma on them, group g + 1 issued before group g's epilogue (bias, LeakyReLU on the accumulator fragments).  Psrc | Pdst
// | Q (and K | V without K/V blocks) leave through the chain's staging tile as whole 256-byte rows; K and V go straight from
// the fragments into the 8-node kv blocks (a quad writes 16 contiguous bytes of a block row, a warp 8 whole block rows).
// Every output element takes the split, products, order and epilogue of the 128-row kernel it replaces.
// P = 3 (bf16x3): two-term h splits and the three leading products.  The K / V blocks are written as full bf16x3 in both
// modes, so the attention of either mode can read them.
#define PJ_CHAINS 2
#define PJ64_W_BYTES (5 * PjCfg<false>::GROUP_BYTES)
#define PJ_OUT_LD 72   // fp32 row stride of the output staging tile (72 % 32 = 8: the fragment stores are conflict-free)

struct __align__(128) PjChainSmem {
  float hs[64 * 64];              // h rows of the next tile (16-byte chunks swizzled, staged_rows_to_a_split3)
  float out[64 * PJ_OUT_LD];      // one group's outputs on their way to proj
};
struct Pj64Smem {
  unsigned char w[PJ64_W_BYTES];
  PjChainSmem ch[PJ_CHAINS];
  float b[320];
  unsigned long long w_bar;
};

template <int P>
__global__ void __launch_bounds__(PJ_CHAINS * 128, 1)
project64_tc_kernel(int n_nodes, eqd_layer_params p, const __grid_constant__ PjConsts cst, const float* __restrict__ h,
                    float* __restrict__ proj, unsigned char* __restrict__ kv, long kv_split_stride) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  Pj64Smem& S = *reinterpret_cast<Pj64Smem*>(smem_raw);
  const int tid = threadIdx.x, wgi = tid >> 7, t = tid & 127, lane = t & 31;
  PjChainSmem& W = S.ch[wgi];
  const int bar = 1 + wgi;   // this chain's named barrier
  const int ntiles = (n_nodes + 63) / 64, tstride = gridDim.x * PJ_CHAINS;
  if (tid == 0) {
    mbar_init(&S.w_bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    mbar_expect_tx(&S.w_bar, PJ64_W_BYTES);
    bulk_g2s(S.w, p.w_proj_tc, PJ64_W_BYTES, &S.w_bar);
  }
  for (int i = tid; i < 320; i += PJ_CHAINS * 128) S.b[i] = cst.b[i];
  __syncthreads();
  const unsigned w_saddr = smem_u32(S.w);
  const float slope = p.leaky_slope;
  // accumulator-fragment rows of this thread: fr0 and fr0 + 8; columns 8 j + fc + {0, 1}, j = 0..7
  const int fr0 = (t >> 5) * 16 + (lane >> 2), fc = 2 * (lane & 3);
  auto stage_h = [&](int tile) { stage_rows64(W.hs, h, EQD_HID, 0, (long)tile * 64, min(64, n_nodes - tile * 64), t); };
  int tile = blockIdx.x * PJ_CHAINS + wgi;
  if (tile < ntiles) stage_h(tile);
  mbar_wait(&S.w_bar, 0);

  for (; tile < ntiles; tile += tstride) {
    const int node0 = tile * 64, nvalid = min(64, n_nodes - node0);
    cp_async_wait<0>();
    wg_barrier(bar);   // this tile's h rows have landed
    unsigned af[3][4][4];
    staged_rows_to_a_split3<P>(W.hs, t, af);
    wg_barrier(bar);   // the staging buffer is free
    if (tile + tstride < ntiles) stage_h(tile + tstride);
    auto group = [&](int grp) {
      return [&, grp](int s, int kb) { return b_desc_ex(w_saddr + grp * PjCfg<false>::GROUP_BYTES + s * PjCfg<false>::SPLIT_BYTES + kb * 2048, 1024, 128); };
    };
    float acc[2][32];
    wg_gemm6_rs_issue<64, 4, 0, false, P>(acc[0], af, group(0), false);
#pragma unroll
    for (int grp = 0; grp < 5; ++grp) {
      float (&d)[32] = acc[grp & 1];
      if (grp + 1 < 5) {
        wg_gemm6_rs_issue<64, 4, 0, false, P>(acc[(grp + 1) & 1], af, group(grp + 1), false);
        wg_mma_wait<1>(d);
      } else {
        wg_mma_wait(d);
      }
      const bool act = (grp == 2 || grp == 3);        // Q, K carry the LeakyReLU
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float2 bj = *reinterpret_cast<const float2*>(&S.b[grp * 64 + 8 * j + fc]);
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          float& x0 = d[4 * j + 2 * hh];
          float& x1 = d[4 * j + 2 * hh + 1];
          x0 = x0 + bj.x;
          x1 = x1 + bj.y;
          if (act) {
            x0 = lrelu(x0, slope);
            x1 = lrelu(x1, slope);
          }
        }
      }
      if (grp < 3 || kv == nullptr) {   // with K/V blocks requested nobody reads the fp32 K / V columns
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
          for (int hh = 0; hh < 2; ++hh)
            *reinterpret_cast<float2*>(W.out + (fr0 + 8 * hh) * PJ_OUT_LD + 8 * j + fc) =
                make_float2(d[4 * j + 2 * hh], d[4 * j + 2 * hh + 1]);
        wg_barrier(bar);
        // 16 lanes per 256-byte row, 8 rows per pass
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int row = i * 8 + (t >> 4), c4 = t & 15;
          if (row < nvalid)
            *reinterpret_cast<float4*>(proj + (long)(node0 + row) * 320 + grp * 64 + 4 * c4) =
                *reinterpret_cast<const float4*>(W.out + row * PJ_OUT_LD + 4 * c4);
        }
        wg_barrier(bar);   // the staging tile is free for the next group
      } else {
        // kv[which][split][n/8][d/8][n%8][d%8]: channels (8 j + fc, + 1) of a row are one 4-byte word per split
        unsigned char* base = kv + (long)(grp - 3) * 3 * kv_split_stride;
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int row = fr0 + 8 * hh, node = node0 + row;
          if (row < nvalid) {
            unsigned char* nb = base + (long)(node >> 3) * 1024 + (node & 7) * 16 + fc * 2;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              unsigned w0, w1, w2;
              split3_pair(d[4 * j + 2 * hh], d[4 * j + 2 * hh + 1], w0, w1, w2);
              *reinterpret_cast<unsigned*>(nb + j * 128) = w0;
              *reinterpret_cast<unsigned*>(nb + kv_split_stride + j * 128) = w1;
              *reinterpret_cast<unsigned*>(nb + 2 * kv_split_stride + j * 128) = w2;
            }
          }
        }
      }
    }
  }
  cp_async_wait<0>();
}

// fp32 K / V columns of a projection buffer -> bf16x3 8-node blocks (used after the FFMA layer-0 node stage)
__global__ void kv_blocks_kernel(int n_nodes, const float* __restrict__ proj, int pw, int koff, int voff,
                                 unsigned char* __restrict__ kv, long kv_split_stride) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;  // (node, which, half)
  int node = idx >> 2, which = (idx >> 1) & 1, half = idx & 1;
  if (node >= n_nodes) return;
  const float4* src = reinterpret_cast<const float4*>(proj + (long)node * pw + (which ? voff : koff) + half * 32);
  float v[32];
#pragma unroll
  for (int c4 = 0; c4 < 8; ++c4) {
    float4 t = src[c4];
    v[c4 * 4] = t.x; v[c4 * 4 + 1] = t.y; v[c4 * 4 + 2] = t.z; v[c4 * 4 + 3] = t.w;
  }
  store_kv_blocks(kv + (long)which * 3 * kv_split_stride, kv_split_stride, node, half, v);
}

}  // namespace eqd

extern "C" size_t eqd_kv_blocks_bytes(int32_t n_nodes) {
  // [which 2][split 3][ceil(n/8) + 8 pad groups][1024 B]; the pad groups must be zero (they feed P.V as 0 x V)
  return (size_t)6 * ((size_t)(n_nodes + 7) / 8 + 8) * 1024;
}

template <bool L0>
static int launch_project_tc(const eqd_graph* g, const eqd_layer* p_l, const float* h, int ldh, float* proj, int pw,
                             void* kv, float* x5, void* stream) {
  const eqd_layer_params* p = &p_l->dev;
  if (!(p->leaky_slope >= 0.f && p->leaky_slope <= 1.f)) return EQD_ERR_UNSUPPORTED;  // lrelu() = max(v, slope*v)
  if (!p->w_proj_tc || (reinterpret_cast<uintptr_t>(p->w_proj_tc) & 15)) return EQD_ERR_BAD_ARG;
  if (g->n_nodes <= 0) return EQD_OK;
  eqd::PjConsts cst;
  memset(&cst, 0, sizeof(cst));
  memcpy(&cst, p_l->consts.proj_bias, 320 * sizeof(float));
  int ntiles = (g->n_nodes + eqd::PjCfg<L0>::R - 1) / eqd::PjCfg<L0>::R;
  size_t smem = sizeof(eqd::PjSmem<L0>) + 128;
  EQD_SET_SMEM((eqd::project_tc_kernel<L0>), smem);
  int grid = ntiles < EQD_SMS ? ntiles : EQD_SMS;
  long split_stride = (long)((g->n_nodes + 7) / 8 + 8) * 1024;
  eqd::project_tc_kernel<L0><<<grid, eqd::PjCfg<L0>::THREADS, smem, (cudaStream_t)stream>>>(
      g->n_nodes, *p, cst, h, ldh, proj, pw, reinterpret_cast<unsigned char*>(kv), split_stride, x5);
  EQD_CUDA_LAUNCH_CHECK();
  return EQD_OK;
}

template <int P>
static int launch_project64_tc(const eqd_graph* g, const eqd_layer* p_l, const float* h, float* proj, void* kv,
                               void* stream) {
  eqd::PjConsts cst;
  memset(&cst, 0, sizeof(cst));
  memcpy(&cst, p_l->consts.proj_bias, 320 * sizeof(float));
  const int ntiles = (g->n_nodes + 63) / 64;
  const size_t smem = sizeof(eqd::Pj64Smem) + 128;
  EQD_SET_SMEM(eqd::project64_tc_kernel<P>, smem);
  int grid = (ntiles + PJ_CHAINS - 1) / PJ_CHAINS;
  if (grid > EQD_SMS) grid = EQD_SMS;
  const long split_stride = (long)((g->n_nodes + 7) / 8 + 8) * 1024;
  eqd::project64_tc_kernel<P><<<grid, PJ_CHAINS * 128, smem, (cudaStream_t)stream>>>(
      g->n_nodes, p_l->dev, cst, h, proj, reinterpret_cast<unsigned char*>(kv), split_stride);
  EQD_CUDA_LAUNCH_CHECK();
  return EQD_OK;
}

extern "C" int eqd_project_tc(const eqd_graph* g, const eqd_layer* p_l, const float* h, float* proj, void* kv,
                              void* stream) {
  const eqd_layer_params* p = p_l ? &p_l->dev : nullptr;
  if (!g || !p || !h || !proj) return EQD_ERR_BAD_ARG;
  if (p->dh != 64 || p->dhp != 64) return EQD_ERR_UNSUPPORTED;
  if (!(p->leaky_slope >= 0.f && p->leaky_slope <= 1.f)) return EQD_ERR_UNSUPPORTED;  // lrelu() = max(v, slope*v)
  const int products = eqd_mma_products(p);
  if (!products) return EQD_ERR_UNSUPPORTED;
  if (!p->w_proj_tc || (reinterpret_cast<uintptr_t>(p->w_proj_tc) & 15)) return EQD_ERR_BAD_ARG;
  if (g->n_nodes <= 0) return EQD_OK;
  return products == 3 ? launch_project64_tc<3>(g, p_l, h, proj, kv, stream)
                       : launch_project64_tc<6>(g, p_l, h, proj, kv, stream);
}

extern "C" int eqd_project_tc0(const eqd_graph* g, const eqd_layer* p_l, const float* h0, float* proj, void* kv,
                               float* x5, void* stream) {
  const eqd_layer_params* p = p_l ? &p_l->dev : nullptr;
  if (!g || !p || !h0 || !proj || !kv || !x5) return EQD_ERR_BAD_ARG;
  if (p->dh != 69 || p->dhp != 72 || !eqd_mma_products(p)) return EQD_ERR_UNSUPPORTED;
  return launch_project_tc<true>(g, p_l, h0, EQD_H0_PAD, proj, 128 + 3 * 72, kv, x5, stream);
}

extern "C" int eqd_kv_blocks(const eqd_graph* g, const float* proj, int32_t pw, int32_t koff, int32_t voff, void* kv,
                             void* stream) {
  if (!g || !proj || !kv) return EQD_ERR_BAD_ARG;
  if (g->n_nodes <= 0) return EQD_OK;
  long split_stride = (long)((g->n_nodes + 7) / 8 + 8) * 1024;
  int total = g->n_nodes * 4;
  eqd::kv_blocks_kernel<<<(total + 255) / 256, 256, 0, (cudaStream_t)stream>>>(g->n_nodes, proj, pw, koff, voff,
                                                                                reinterpret_cast<unsigned char*>(kv), split_stride);
  EQD_CUDA_LAUNCH_CHECK();
  return EQD_OK;
}
