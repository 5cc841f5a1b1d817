// Training minibatches gathered from a device-resident pair archive (eqd_assemble_batch, include/eqd_iegmn.h): the
// device replacement of PairArchive.batch -> hetero_graph.batch_pairs -> .to(dev) -> GraphPlan / PocketBatch, plus the
// reference's per-sample random ligand pose (UniformRotation_Translation, src/utils/protein_utils.py:15-23, applied in
// db5_data.py __getitem__).  One CTA row (blockIdx.y) per protein segment of the batch, blockIdx.x strides over the
// segment's rows.  A gather: every byte is read once and written once; the edge features, 27 floats per row and so at
// any 4-float phase in both the archive and the batch, move as aligned 16-byte vectors re-phased in registers.
#include <algorithm>

#include "common.cuh"
#include "philox.cuh"

namespace eqd {

#define BA_THREADS 256

// 53-bit uniform in [0, 1) from two 32-bit words
__device__ __forceinline__ double u01(uint32_t hi, uint32_t lo) {
  return ((double)(hi >> 5) * 67108864.0 + (double)(lo >> 6)) * (1.0 / 9007199254740992.0);
}

// The law of synthetic.random_rigid: q = 4 normals normalised, R(q); t = (3 normals normalised) x U(0, interval).
// Normals by Box-Muller; all in fp64.  rt = R [9] row-major, t [3].
__device__ void draw_rigid(uint64_t seed, uint64_t step, uint32_t slot, double interval, double* rt) {
  const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
  double u[10];
#pragma unroll
  for (int d = 0; d < 5; ++d) {
    const uint4 r = philox4x32_10(make_uint4(slot, (uint32_t)d, (uint32_t)step, (uint32_t)(step >> 32)), key);
    u[2 * d] = u01(r.x, r.y);
    u[2 * d + 1] = u01(r.z, r.w);
  }
  double z[8];
#pragma unroll
  for (int p = 0; p < 4; ++p) {
    const double rad = sqrt(-2.0 * log(1.0 - u[2 * p]));      // 1 - u in (0, 1]
    double sn, cs;
    sincospi(2.0 * u[2 * p + 1], &sn, &cs);
    z[2 * p] = rad * cs;
    z[2 * p + 1] = rad * sn;
  }
  const double qn = rsqrt(z[0] * z[0] + z[1] * z[1] + z[2] * z[2] + z[3] * z[3]);
  const double w = z[0] * qn, a = z[1] * qn, b = z[2] * qn, c = z[3] * qn;
  rt[0] = 1.0 - 2.0 * (b * b + c * c); rt[1] = 2.0 * (a * b - c * w);       rt[2] = 2.0 * (a * c + b * w);
  rt[3] = 2.0 * (a * b + c * w);       rt[4] = 1.0 - 2.0 * (a * a + c * c); rt[5] = 2.0 * (b * c - a * w);
  rt[6] = 2.0 * (a * c - b * w);       rt[7] = 2.0 * (b * c + a * w);       rt[8] = 1.0 - 2.0 * (a * a + b * b);
  const double len = u[8] * interval / sqrt(z[4] * z[4] + z[5] * z[5] + z[6] * z[6]);
  rt[9] = z[4] * len; rt[10] = z[5] * len; rt[11] = z[6] * len;
}

// {w[r], .., w[r+3]} of the 8 floats w = (v0, v1); r is uniform across the CTA
__device__ __forceinline__ float4 rephase(float4 v0, float4 v1, int r) {
  switch (r) {
    case 1: return make_float4(v0.y, v0.z, v0.w, v1.x);
    case 2: return make_float4(v0.z, v0.w, v1.x, v1.y);
    case 3: return make_float4(v0.w, v1.x, v1.y, v1.z);
    default: return v0;
  }
}

__device__ __forceinline__ void pose3(const double* rt, const double* cen, const float* in, float* out) {
  const double d0 = (double)in[0] - cen[0], d1 = (double)in[1] - cen[1], d2 = (double)in[2] - cen[2];
#pragma unroll
  for (int q = 0; q < 3; ++q) out[q] = (float)(rt[q * 3] * d0 + rt[q * 3 + 1] * d1 + rt[q * 3 + 2] * d2 + rt[9 + q]);
}

// min 3 CTAs / SM: 79 registers, no spills (the fp64 pose draw of thread 0 is what needs them)
__global__ void __launch_bounds__(BA_THREADS, 3)
assemble_batch_kernel(const eqd_pair_archive a, const eqd_batch_out o, const int32_t* __restrict__ offsets, int B,
                      uint64_t seed, uint64_t step, int slot0, double interval, int repose) {
  const int s = blockIdx.y;
  const bool lig = s < B;
  const int b = lig ? s : s - B;
  const int32_t* node_off = offsets + B;
  const int32_t* edge_off = node_off + 2 * B + 1;
  const int32_t* pocket_off = edge_off + 2 * B + 1;
  const int32_t* tile_off = pocket_off + B + 1;
  const long i = offsets[b];
  const int n_out0 = node_off[s], nn = node_off[s + 1] - n_out0, N_l = node_off[B];
  const int e_out0 = edge_off[s], ne = edge_off[s + 1] - e_out0;
  const long n_in0 = (lig ? a.lig_node_ptr : a.rec_node_ptr)[i];
  const long e_in0 = (lig ? a.lig_edge_ptr : a.rec_edge_ptr)[i];
  const int t0 = blockIdx.x * BA_THREADS + threadIdx.x, nt = gridDim.x * BA_THREADS;

  __shared__ double rt[12];
  __shared__ double cen[3];
  if (lig) {
    if (threadIdx.x == 0) {
      if (repose) {
        draw_rigid(seed, step, (uint32_t)(slot0 + b), interval, rt);
      } else {
        for (int q = 0; q < 12; ++q) rt[q] = (q == 0 || q == 4 || q == 8) ? 1.0 : 0.0;
      }
      for (int q = 0; q < 3; ++q) cen[q] = a.lig_centroid[i * 3 + q];
    }
    __syncthreads();
    if (blockIdx.x == 0 && threadIdx.x < 12) {
      if (threadIdx.x < 9) o.rot[(long)b * 9 + threadIdx.x] = rt[threadIdx.x];
      else o.trans[(long)b * 3 + threadIdx.x - 9] = rt[threadIdx.x];
    }
  }
  if (t0 == 0) {
    o.seg_ptr[s] = n_out0;
    if (lig) o.pocket_ptr[b] = pocket_off[b];
    if (s == 2 * B - 1) {
      o.seg_ptr[2 * B] = node_off[2 * B];
      o.row_ptr[node_off[2 * B]] = edge_off[2 * B];
      o.pocket_ptr[B] = pocket_off[B];
    }
  }
  for (int t = tile_off[s] + t0; t < tile_off[s + 1]; t += nt) {
    o.node_tiles[2 * t] = s;
    o.node_tiles[2 * t + 1] = n_out0 + EQD_TILE_ROWS * (t - tile_off[s]);
  }

  // ---- nodes ---------------------------------------------------------------------------------------------------------
  const uint8_t* res = lig ? a.lig_res_feat : a.rec_res_feat;
  const float* xin = lig ? a.lig_x : a.rec_x;
  const float* mu = lig ? a.lig_mu_r_norm : a.rec_mu_r_norm;
  const int32_t* dst = (lig ? a.lig_dst : a.rec_dst) + e_in0;
  for (int j = t0; j < nn; j += nt) {
    const long an = n_in0 + j, on = n_out0 + j;
    o.res_feat[on] = (float)res[an];
#pragma unroll
    for (int q = 0; q < 3; ++q) o.x[on * 3 + q] = xin[an * 3 + q];
#pragma unroll
    for (int q = 0; q < 5; ++q) o.mu_r_norm[on * 5 + q] = mu[an * 5 + q];
    int lo = 0, hi = ne;                 // row_ptr = first edge of the segment whose destination is >= j
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (dst[mid] < j) lo = mid + 1;
      else hi = mid;
    }
    o.row_ptr[on] = e_out0 + lo;
    if (lig) {
      if (repose) pose3(rt, cen, xin + an * 3, o.new_x + on * 3);
      else
        for (int q = 0; q < 3; ++q) o.new_x[on * 3 + q] = a.lig_new_x[an * 3 + q];
      for (int q = 0; q < 3; ++q) o.bound_lig[on * 3 + q] = a.bound_lig[an * 3 + q];
    } else {
      for (int q = 0; q < 3; ++q) o.bound_rec[(on - N_l) * 3 + q] = a.bound_rec[an * 3 + q];
    }
  }

  // ---- pocket points (per pair: in the ligand segment) ----------------------------------------------------------------
  if (lig) {
    const long p_in0 = a.pocket_ptr[i];
    const int p_out0 = pocket_off[b], np = pocket_off[b + 1] - p_out0;
    for (int k = t0; k < np; k += nt) {
      const float* pin = a.pocket_coors + (p_in0 + k) * 3;
      const long po = (long)(p_out0 + k) * 3;
      for (int q = 0; q < 3; ++q) o.pocket_rec[po + q] = pin[q];
      if (repose) pose3(rt, cen, pin, o.pocket_lig + po);
      else
        for (int q = 0; q < 3; ++q) o.pocket_lig[po + q] = pin[q];
    }
  }

  // ---- edge ids, renumbered to batch nodes ----------------------------------------------------------------------------
  const int32_t* src = (lig ? a.lig_src : a.rec_src) + e_in0;
  for (int k = t0; k < ne; k += nt) {
    o.col_src[e_out0 + k] = src[k] + n_out0;
    o.edge_dst[e_out0 + k] = dst[k] + n_out0;
  }

  // ---- edge features: the segment's float range [src_f, src_f + nf) -> [dst_f, dst_f + nf), 16-byte vectors --------------
  const float* he_in = lig ? a.lig_he : a.rec_he;
  float* he_out = lig ? o.he_lig : o.he_rec;
  const long src_f = e_in0 * EQD_EDGE_FEATS, nf = (long)ne * EQD_EDGE_FEATS;
  const long dst_f = (long)(lig ? e_out0 : e_out0 - edge_off[B]) * EQD_EDGE_FEATS;
  const long d_lo = dst_f & ~3L, d_hi = (dst_f + nf + 3) & ~3L;
  const long shift = src_f - dst_f;                        // source float of output float d is d + shift
  const int r = (int)(((shift % 4) + 4) % 4);
  for (long d = d_lo + 4L * t0; d < d_hi; d += 4L * nt) {
    if (d >= dst_f && d + 4 <= dst_f + nf) {
      const long s0 = d + shift - r;                       // 16-byte aligned
      const float4 v0 = __ldg(reinterpret_cast<const float4*>(he_in + s0));
      const float4 v1 = r ? __ldg(reinterpret_cast<const float4*>(he_in + s0 + 4)) : v0;
      *reinterpret_cast<float4*>(he_out + d) = rephase(v0, v1, r);
    } else {                                               // a vector shared with the neighbouring segment
      for (long q = d; q < d + 4; ++q)
        if (q >= dst_f && q < dst_f + nf) he_out[q] = he_in[q + shift];
    }
  }
}

}  // namespace eqd

extern "C" int eqd_assemble_batch(const eqd_pair_archive* archive, int32_t n_batch, const int32_t* offsets,
                                  int32_t max_segment_edges, uint64_t seed, uint64_t step, int32_t slot0,
                                  float translation_interval, int32_t repose, const eqd_batch_out* out, void* stream) {
  if (!archive || !out || !offsets || n_batch < 0 || max_segment_edges < 0 || slot0 < 0) return EQD_ERR_BAD_ARG;
  const eqd_batch_out& o = *out;
  const eqd_pair_archive& a = *archive;
  if (!a.lig_node_ptr || !a.rec_node_ptr || !a.lig_edge_ptr || !a.rec_edge_ptr || !a.pocket_ptr || !a.lig_res_feat ||
      !a.rec_res_feat || !a.lig_x || !a.rec_x || !a.lig_mu_r_norm || !a.rec_mu_r_norm || !a.lig_src || !a.lig_dst ||
      !a.rec_src || !a.rec_dst || !a.lig_he || !a.rec_he || !a.lig_new_x || !a.pocket_coors || !a.bound_lig ||
      !a.bound_rec || !a.lig_centroid)
    return EQD_ERR_BAD_ARG;
  if (!o.res_feat || !o.x || !o.new_x || !o.mu_r_norm || !o.row_ptr || !o.col_src || !o.edge_dst || !o.he_lig || !o.he_rec ||
      !o.seg_ptr ||
      !o.node_tiles || !o.pocket_ptr || !o.pocket_lig || !o.pocket_rec || !o.bound_lig || !o.bound_rec || !o.rot || !o.trans)
    return EQD_ERR_BAD_ARG;
  if (((uintptr_t)a.lig_he | (uintptr_t)a.rec_he | (uintptr_t)o.he_lig | (uintptr_t)o.he_rec) & 15) return EQD_ERR_BAD_ARG;
  if (n_batch == 0) return EQD_OK;
  if (n_batch > 32767) return EQD_ERR_UNSUPPORTED;             // 2B segments on grid y
  const long vec = ((long)max_segment_edges * EQD_EDGE_FEATS + 3) / 4 + 1;
  const unsigned gx = (unsigned)std::min<long>(std::max<long>((vec + BA_THREADS - 1) / BA_THREADS, 1L), 1024L);
  eqd::assemble_batch_kernel<<<dim3(gx, 2 * n_batch), BA_THREADS, 0, (cudaStream_t)stream>>>(
      a, o, offsets, n_batch, seed, step, slot0, (double)translation_interval, repose);
  EQD_CUDA_LAUNCH_CHECK();
  return EQD_OK;
}
