// The start of an edge tile, shared by the edge stage (edge_stage.cu) and its backward (bwd_edge.cu), which recomputes
// the forward's per-edge activations: the layer's weights in shared memory, the per-edge geometry and RBFs, the original
// edge features and z1 = Psrc[src] + Pdst[dst] + W1e [he | rbf] with its dropout.  Both kernels run it on a contiguous
// edge range [e0, e0 + ne), ne <= 128: the forward's edges of a tile of destination nodes, the backward's 128
// consecutive edges.
#pragma once
#include "common.cuh"
#include "philox.cuh"

namespace eqd {

#define EDGE_K1 44    // 27 he + 15 rbf + 2 zero
#define EDGE_LD1 48   // smem row stride of the [he|rbf] operand
#define EDGE_LD 68    // smem row stride of 64-wide operands

// Shared-memory prefix of both edge kernels.
struct EdgeTileSmem {
  float w1[EDGE_K1 * 64];       // k-major [he|rbf] rows of edge_mlp.0
  float w2[64 * 64];            // k-major edge_mlp.4
  float w3[64 * 64];            // k-major coors_mlp.0
  float ln_g[64], ln_b[64], b2[64], b3[64], w4[64];
  float cln_g[64], cln_b[64];   // coors_mlp.3 (CLN only)
  double xrel[EQD_TM * 3];
  int src[EQD_TM], dst[EQD_TM];
};

// The layer's weights and vectors -> s (CLN: also coors_mlp.3 of `nm`).  All 128 threads; the caller synchronises.
template <bool CLN>
__device__ __forceinline__ void edge_tile_weights(EdgeTileSmem& s, const eqd_layer_params& p, const eqd_layer_norms& nm,
                                                  int tid) {
  for (int i = tid; i < EDGE_K1 * 64 / 4; i += EQD_THREADS)
    reinterpret_cast<float4*>(s.w1)[i] = reinterpret_cast<const float4*>(p.w_edge1)[i];
  for (int i = tid; i < 64 * 64 / 4; i += EQD_THREADS) {
    reinterpret_cast<float4*>(s.w2)[i] = reinterpret_cast<const float4*>(p.w_edge2)[i];
    reinterpret_cast<float4*>(s.w3)[i] = reinterpret_cast<const float4*>(p.w_coor1)[i];
  }
  if (tid < 64) {
    s.ln_g[tid] = p.edge_ln_g[tid];
    s.ln_b[tid] = p.edge_ln_b[tid];
    s.b2[tid] = p.b_edge2[tid];
    s.b3[tid] = p.b_coor1[tid];
    s.w4[tid] = p.w_coor2[tid];
  }
  if (CLN && tid < 64) {
    s.cln_g[tid] = nm.coors_ln_g[tid];
    s.cln_b[tid] = nm.coors_ln_b[tid];
  }
}

// Per-edge inputs of edges [e0, e0 + ne), thread t <-> edge e0 + t: s.src / s.dst (-1 past ne), x_rel = x[src] - x[dst]
// in fp64 (u_sub_v :204-205) and row t of ein (row stride EDGE_LD1) = [he | 15 RBFs exp(-d^2 / 1.5^q) (:208-210) | 0 0],
// all 0 past ne.  The tile's he rows are contiguous in one of he_lig / he_rec.  All 128 threads; the caller
// synchronises.
__device__ __forceinline__ void edge_tile_inputs(EdgeTileSmem& s, float* __restrict__ ein, const eqd_graph& g,
                                                 const double* __restrict__ x_in, int e0, int ne, int tid) {
  float* row = ein + tid * EDGE_LD1;
  if (tid < ne) {
    const int e = e0 + tid;
    const int sn = g.col_src[e], dn = g.edge_dst[e];
    s.src[tid] = sn;
    s.dst[tid] = dn;
    const double rx = x_in[(long)sn * 3 + 0] - x_in[(long)dn * 3 + 0];
    const double ry = x_in[(long)sn * 3 + 1] - x_in[(long)dn * 3 + 1];
    const double rz = x_in[(long)sn * 3 + 2] - x_in[(long)dn * 3 + 2];
    s.xrel[tid * 3 + 0] = rx;
    s.xrel[tid * 3 + 1] = ry;
    s.xrel[tid * 3 + 2] = rz;
    const float d2 = (float)(rx * rx + ry * ry + rz * rz);
    float sigma = 1.f;
#pragma unroll
    for (int q = 0; q < EQD_N_RBF; ++q) {
      row[EQD_EDGE_FEATS + q] = expf(-d2 / sigma);
      sigma *= 1.5f;
    }
  } else {
    s.src[tid] = -1;
    s.dst[tid] = -1;
#pragma unroll
    for (int q = 0; q < EQD_N_RBF; ++q) row[EQD_EDGE_FEATS + q] = 0.f;
  }
  row[42] = 0.f;
  row[43] = 0.f;
  for (int idx = tid; idx < EQD_TM * EQD_EDGE_FEATS; idx += EQD_THREADS) {
    int r = idx / EQD_EDGE_FEATS, k = idx - r * EQD_EDGE_FEATS;
    float v = 0.f;
    if (r < ne) {
      int e = e0 + r;
      v = e < g.n_lig_edges ? g.he_lig[(long)e * EQD_EDGE_FEATS + k]
                            : g.he_rec[(long)(e - g.n_lig_edges) * EQD_EDGE_FEATS + k];
    }
    ein[r * EDGE_LD1 + k] = v;
  }
}

// z1 of edge_mlp.0 on this thread's 8 rows of the tile: the gathered node projections Psrc[src] + Pdst[dst] (+bias) of
// proj (row width pw), 0 for rows past the tile, plus the [he|rbf] GEMM on ein; DROP: dropout site 0 of `dr`.
template <bool DROP>
__device__ __forceinline__ void edge_tile_z1(float (&acc)[8][8], float (&accx)[8], const EdgeTileSmem& s,
                                             const float* ein, const float* __restrict__ proj, int pw,
                                             const eqd_dropout& dr, int e0, int ty, int tx) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    int r = ty * 8 + i;
    int sn = s.src[r], dn = s.dst[r];
    if (sn >= 0) {
      const float* ps = proj + (long)sn * pw + tx * 4;       // Psrc row
      const float* pd = proj + (long)dn * pw + 64 + tx * 4;  // Pdst row (+bias)
      float4 a0 = *reinterpret_cast<const float4*>(ps), a1 = *reinterpret_cast<const float4*>(ps + 32);
      float4 b0 = *reinterpret_cast<const float4*>(pd), b1 = *reinterpret_cast<const float4*>(pd + 32);
      acc[i][0] = a0.x + b0.x; acc[i][1] = a0.y + b0.y; acc[i][2] = a0.z + b0.z; acc[i][3] = a0.w + b0.w;
      acc[i][4] = a1.x + b1.x; acc[i][5] = a1.y + b1.y; acc[i][6] = a1.z + b1.z; acc[i][7] = a1.w + b1.w;
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
    }
  }
  gemm_nn<false>(acc, accx, ein + ty * 8 * EDGE_LD1, EDGE_LD1, s.w1, 64, EDGE_K1, tx);
  if (DROP) dropout_tile<false>(acc, accx, dr, 0, e0 + ty * 8, tx);
}

}  // namespace eqd
