// Training losses of the reference on the device (SURVEY 8f rank 1), one CTA per protein pair, with their gradients:
//   * per-pair MSE of the predicted ligand C-alpha coordinates (nn.MSELoss, src/train.py:114)
//   * body-intersection loss (src/train.py:41-49, 131-133): two n x m Gaussian log-sum reductions
//   * pocket OT loss (src/train.py:125-129, src/utils/ot_utils.py:5-29): cost = |P_l - Y_l|^2 + |P_r - Y_r|^2 between the
//     N_pocket pocket points and the K keypoints (num_att_heads, 1..64), EXACT earth mover's distance with uniform marginals.  The reference calls
//     POT's network simplex on the CPU (ot.emd, a D2H/H2D round trip per pair); here the transport LP is solved on the SM
//     by successive shortest augmenting paths with node potentials (primal-dual; Dijkstra on the dense bipartite residual
//     graph, integer flows in units of 1/(N_pocket * K)), which terminates at the LP optimum -- the unique optimal VALUE any
//     exact solver returns.  The plan is a constant for the gradient (ot_utils.py:27): dY = 2 sum_i T_ik (Y_k - P_i).
// Everything in fp64; all reductions in a fixed order.  Restated in oracle/loss_oracle.py.
#include "common.cuh"

namespace eqd {

#define LOSS_THREADS 128
#define OT_MAX_POCKET 1024

__device__ __forceinline__ double block_sum_d(double v, double* sh /*[LOSS_THREADS]*/) {
  __syncthreads();
  sh[threadIdx.x] = v;
  __syncthreads();
  for (int s = LOSS_THREADS / 2; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
    __syncthreads();
  }
  double r = sh[0];
  __syncthreads();
  return r;
}

// parts[b] = {mse, intersection}; dcoors[i] = d (mse/B + w_int * inter/B) / d pred_i
__global__ void __launch_bounds__(LOSS_THREADS)
loss_mse_intersection_kernel(eqd_graph g, const float* __restrict__ pred, const float* __restrict__ tgt_lig,
                             const float* __restrict__ rec, double sigma, double surface_ct, double w_int,
                             double* __restrict__ wrec /*[N_r] scratch*/, double* __restrict__ parts,
                             float* __restrict__ dcoors) {
  __shared__ double sh[LOSS_THREADS];
  const int b = blockIdx.x, B = g.n_pairs, tid = threadIdx.x;
  const int l0 = g.seg_ptr[b], l1 = g.seg_ptr[b + 1];
  const int r0 = g.seg_ptr[B + b] - g.n_lig_nodes, r1 = g.seg_ptr[B + b + 1] - g.n_lig_nodes;   // receptor-local ids
  const int nl = l1 - l0, nr = r1 - r0;
  const double invB = 1.0 / (double)B;
  // pass B first: per receptor point, S_i = 1e-3 + sum_j exp(-|y_i - l_j|^2 / sigma) -> active weight
  double t2 = 0.0;
  for (int i = r0 + tid; i < r1; i += LOSS_THREADS) {
    const double yx = rec[(long)i * 3], yy = rec[(long)i * 3 + 1], yz = rec[(long)i * 3 + 2];
    double S = 1e-3;
    for (int j = l0; j < l1; ++j) {
      const double dx = yx - pred[(long)j * 3], dy = yy - pred[(long)j * 3 + 1], dz = yz - pred[(long)j * 3 + 2];
      S += exp(-(dx * dx + dy * dy + dz * dz) / sigma);
    }
    const double val = surface_ct + sigma * log(S);       // ct - G_lig(y_i)
    const bool act = val > 0.0;
    t2 += act ? val : 0.0;
    wrec[i] = act ? 1.0 / ((double)nr * S) : 0.0;
  }
  const double term2 = block_sum_d(t2, sh) / (double)(nr > 0 ? nr : 1);
  __threadfence_block();
  __syncthreads();
  double t1 = 0.0, tm = 0.0;
  for (int j = l0 + tid; j < l1; j += LOSS_THREADS) {
    const double px = pred[(long)j * 3], py = pred[(long)j * 3 + 1], pz = pred[(long)j * 3 + 2];
    double S = 1e-3, vx = 0.0, vy = 0.0, vz = 0.0, gx = 0.0, gy = 0.0, gz = 0.0;
    for (int i = r0; i < r1; ++i) {
      const double dx = px - rec[(long)i * 3], dy = py - rec[(long)i * 3 + 1], dz = pz - rec[(long)i * 3 + 2];
      const double e = exp(-(dx * dx + dy * dy + dz * dz) / sigma);
      S += e;
      vx += e * dx; vy += e * dy; vz += e * dz;
      const double w = wrec[i] * e;                         // term 2: d/d l_j = 2 e_ij (y_i - l_j) / (n_r S_i) = -2 w (l_j - y_i)
      gx -= w * dx; gy -= w * dy; gz -= w * dz;
    }
    const double val = surface_ct + sigma * log(S);         // ct - G_rec(l_j)
    const bool act = val > 0.0;
    t1 += act ? val : 0.0;
    const double c1 = act ? -2.0 / ((double)nl * S) : 0.0;  // d(ct - G_rec)/d l_j = -2 sum_i e_i (l_j - r_i) / S
    const double ex = px - tgt_lig[(long)j * 3], ey = py - tgt_lig[(long)j * 3 + 1], ez = pz - tgt_lig[(long)j * 3 + 2];
    tm += ex * ex + ey * ey + ez * ez;
    const double cm = 2.0 / (3.0 * (double)nl);
    dcoors[(long)j * 3 + 0] = (float)(invB * (cm * ex + w_int * (c1 * vx + 2.0 * gx)));
    dcoors[(long)j * 3 + 1] = (float)(invB * (cm * ey + w_int * (c1 * vy + 2.0 * gy)));
    dcoors[(long)j * 3 + 2] = (float)(invB * (cm * ez + w_int * (c1 * vz + 2.0 * gz)));
  }
  const double term1 = block_sum_d(t1, sh) / (double)(nl > 0 ? nl : 1);
  const double mse = block_sum_d(tm, sh) / (3.0 * (double)(nl > 0 ? nl : 1));
  if (tid == 0) {
    parts[(long)b * 4 + 0] = mse;
    parts[(long)b * 4 + 2] = term1 + term2;
  }
}

// Per-CTA state of the transport solver, carved from dynamic shared memory for a pocket capacity `cap` (the largest pocket
// of the batch) and M = K keypoints.  The cost matrix C (fp64, cap x M) and the per-sink source lists (int16) live in shared
// memory when they fit (M = 50: cap <= 310: both; <= 370: C only; <= 870: lists only), else in global memory (L2); flows
// x_ik <= M <= 64 are int8.
struct OtView {
  double *P, *Y, *u, *v, *base_v, *Cm;
  double *Wv, *dsink;          // sink graph: Wv[k][64] = min over the feeders i of sink k of C[i][.] - u[i]; settle distances
  int *excess, *exl, *exq, *stamp, *deficit, *par_k, *par_via, *fl_cnt, *base_i, *ord;
  signed char* xs;
  short *fls, *Wi;             // Wi[k][64] = the feeder that attains Wv (-1: none)
};
#define OT_WLD 64
struct OtLayout {
  size_t bytes;
  int c_smem, fl_smem;
};
__host__ __device__ inline OtLayout ot_layout(int cap, int M) {
  const size_t fixed = (size_t)(cap * 6 + M * 6 + cap + 2 * M + M * OT_WLD + OT_WLD) * 8 +
                       (size_t)(4 * cap + 5 * M + OT_WLD) * 4 + (size_t)M * OT_WLD * 2 + (size_t)cap * M + 256;
  const size_t cbytes = (size_t)cap * M * 8, fbytes = (size_t)cap * M * 2;
  const size_t lim = 227 * 1024 - 2048;      // static shared memory of the kernel is ~1.5 KB
  OtLayout L;
  L.c_smem = fixed + cbytes <= lim;
  L.fl_smem = fixed + (L.c_smem ? cbytes : 0) + fbytes <= lim;
  L.bytes = fixed + (L.c_smem ? cbytes : 0) + (L.fl_smem ? fbytes : 0);
  return L;
}
__device__ inline OtView ot_carve(unsigned char* base, int cap, int M, const OtLayout& L, double* c_global, short* fl_global) {
  OtView s;
  double* d = reinterpret_cast<double*>(base);
  s.P = d; d += cap * 6;
  s.Y = d; d += M * 6;
  s.u = d; d += cap;
  s.v = d; d += M;
  s.base_v = d; d += M;
  s.Wv = d; d += M * OT_WLD;
  s.dsink = d; d += OT_WLD;
  if (L.c_smem) { s.Cm = d; d += (size_t)cap * M; } else s.Cm = c_global;
  int* i = reinterpret_cast<int*>(d);
  s.excess = i; i += cap;
  s.exl = i; i += cap;
  s.exq = i; i += cap;
  s.stamp = i; i += cap;
  s.deficit = i; i += M;
  s.par_k = i; i += M;
  s.par_via = i; i += M;
  s.fl_cnt = i; i += M;
  s.base_i = i; i += M;
  s.ord = i; i += OT_WLD;
  short* h = reinterpret_cast<short*>(i);
  s.Wi = h; h += M * OT_WLD;
  if (L.fl_smem) { s.fls = h; h += (size_t)cap * M; } else s.fls = fl_global;
  s.xs = reinterpret_cast<signed char*>(h);
  return s;
}

// lexicographic (value, index) minimum over the warp of non-negative doubles: the bit pattern of a non-negative double is
// monotone as a 64-bit unsigned integer, so three 32-bit warp reductions replace five rounds of 64-bit shuffles
__device__ __forceinline__ void warp_argmin(double& v, int& k) {
  const unsigned long long b = (unsigned long long)__double_as_longlong(v);
  const unsigned hi = (unsigned)(b >> 32), lo = (unsigned)b;
  const unsigned mh = __reduce_min_sync(0xffffffffu, hi);
  const unsigned ml = __reduce_min_sync(0xffffffffu, hi == mh ? lo : 0xffffffffu);
  const unsigned mk = __reduce_min_sync(0xffffffffu, (hi == mh && lo == ml) ? (unsigned)k : 0xffffffffu);
  v = __longlong_as_double((long long)(((unsigned long long)mh << 32) | ml));
  k = (int)mk;
}

// One CTA per pair: successive shortest augmenting paths with node potentials on the transport problem scaled to integers
// (supply M = K per pocket point, demand n per keypoint, n * M units in all).
//   * Forward arcs form a complete bipartite graph and backward arcs (k -> i, x_ik > 0) have reduced cost 0 (complementary
//     slackness), so the search only has to SETTLE SINKS; it runs on the sink graph (M <= 64 nodes): a settled sink k reaches the
//     sources that feed it for free, hence every sink k' at  W[k][k'] - v[k'],  W[k][k'] = min over the feeders i of k of
//     (C[i][k'] - u[i]).  Every augmentation starts with all four warps rebuilding W (M x M minima over the ~n + M
//     non-zero flows, independent loads); the Dijkstra itself then runs in warp 0 out of registers -- lane l owns sinks l
//     and l + 32 -- with one shared-memory row read per settled sink.  All unsettled sinks at the current minimum distance
//     are settled in one round (arc lengths >= 0; with potentials most of the search happens at distance 0).
//   * Potentials are kept modulo the common shift of an augmentation (u += D everywhere, v -= D everywhere leaves every
//     reduced cost unchanged): only the sources feeding settled sinks (u += D - d_sink, first sink in settle order) and the
//     settled sinks (v -= D - d) are touched; the sources that still have excess all sit at distance 0 and share ONE lazy
//     offset, so their contribution to the initial sink distances, base[k] = min_i (C_ik - u_i), changes only when the
//     minimiser leaves the excess set.
//   * All minima are lexicographic in (value, index): the plan does not depend on list or lane order.
// The final flows are written to flow[(p0 + i) * M + k] (int32, global).
__global__ void __launch_bounds__(LOSS_THREADS)
ot_emd_kernel(int n_pairs, int cap, int M, const int* __restrict__ pocket_ptr, const float* __restrict__ pocket_lig,
              const float* __restrict__ pocket_rec, const double* __restrict__ keypts, double w_ot,
              int* __restrict__ flow, short* __restrict__ lists_g, double* __restrict__ cost_g, double* __restrict__ parts,
              double* __restrict__ dkeypts, int* __restrict__ err) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int b = blockIdx.x, tid = threadIdx.x, B = n_pairs;
  const int p0 = pocket_ptr[b], n = pocket_ptr[b + 1] - p0;
  const OtLayout L = ot_layout(cap, M);
  const OtView s = ot_carve(smem_raw, cap, M, L, cost_g + (long)p0 * M, lists_g + (long)p0 * M);
  __shared__ double red[LOSS_THREADS];
  __shared__ int redi[LOSS_THREADS];
  if (n <= 0 || n > cap) {
    if (tid == 0) {
      parts[(long)b * 4 + 1] = 0.0;
      if (n > cap) atomicOr(err, 1);
    }
    for (int o = tid; o < 2 * M * 3; o += LOSS_THREADS) {
      const int side = o / (M * 3), rem = o - side * M * 3;
      dkeypts[((long)(side == 0 ? b : B + b) * M) * 3 + rem] = 0.0;
    }
    return;
  }
  for (int o = tid; o < n * 3; o += LOSS_THREADS) {
    const int i = o / 3, c = o - i * 3;
    s.P[i * 6 + c] = (double)pocket_lig[(long)(p0 + i) * 3 + c];
    s.P[i * 6 + 3 + c] = (double)pocket_rec[(long)(p0 + i) * 3 + c];
  }
  for (int o = tid; o < M * 3; o += LOSS_THREADS) {
    const int k = o / 3, c = o - k * 3;
    s.Y[k * 6 + c] = keypts[((long)b * M + k) * 3 + c];
    s.Y[k * 6 + 3 + c] = keypts[((long)(B + b) * M + k) * 3 + c];
  }
  __syncthreads();
  for (int o = tid; o < n * M; o += LOSS_THREADS) {      // cost matrix, once
    const int i = o / M, k = o - i * M;
    double c = 0.0;
#pragma unroll
    for (int q = 0; q < 6; ++q) {
      const double d = s.P[i * 6 + q] - s.Y[k * 6 + q];
      c = fma(d, d, c);
    }
    s.Cm[o] = c;
    s.xs[o] = 0;
  }
  __syncthreads();
  for (int i = tid; i < n; i += LOSS_THREADS) {          // u_i = min_k C_ik, v = 0: all reduced costs >= 0
    double mn = INFINITY;
    for (int k = 0; k < M; ++k) mn = fmin(mn, s.Cm[i * M + k]);
    s.u[i] = mn;                 // for a source WITH excess the true potential is u[i] + u_ex_off (lazy common shift)
    s.excess[i] = M;
    s.exl[i] = i;
    s.exq[i] = i;
    s.stamp[i] = 0;
  }
  if (tid < M) { s.v[tid] = 0.0; s.deficit[tid] = n; s.fl_cnt[tid] = 0; }
  __syncthreads();
  {   // base[k] = min over the sources with excess of (C_ik - u_i): two threads per sink, merged lexicographically
    const int k = tid & 63, part = tid >> 6;
    double best = INFINITY;
    int bi = 0x7fffffff;
    if (k < M)
      for (int q = part; q < n; q += 2) {
        const double c = s.Cm[q * M + k] - s.u[q];
        if (c < best || (c == best && q < bi)) { best = c; bi = q; }
      }
    red[tid] = best;
    redi[tid] = bi;
    __syncthreads();
    if (tid < M) {
      const double o2 = red[tid + 64];
      const int i2 = redi[tid + 64];
      if (o2 < best || (o2 == best && i2 < bi)) { best = o2; bi = i2; }
      s.base_v[tid] = best;
      s.base_i[tid] = bi;
    }
    __syncthreads();
  }
  long n_aug = 0, n_pop = 0;
  __shared__ int sh_mass, sh_fail;
  {
    const int lane = tid & 31, warp = tid >> 5;
    const int k0 = lane, k1 = lane + 32;               // the two sinks a lane owns (each valid iff < M)
    const bool has0 = k0 < M, has1 = k1 < M;
    int mass = n * M, nex = n, epoch = 0, fail = 0;    // solver state: warp 0
    double u_ex_off = 0.0;
    const long max_aug = 64L * (n + M) + 1024;
    auto X = [&](int i, int k) -> int { return (int)s.xs[i * M + k]; };
    if (tid == 0) { sh_mass = mass; sh_fail = 0; }
    __syncthreads();
    while (sh_mass > 0 && !sh_fail && n_aug < max_aug) {
      ++n_aug;
      ++epoch;
      // ---- A (all warps): the sink graph.  A settled sink k reaches, at no cost, the sources that feed it (backward arcs of
      // reduced cost 0), and through source i every sink k' at C[i][k'] - u[i] - v[k']: its outgoing arc lengths are
      // W[k][k'] - v[k'] with W[k][k'] = min over the feeders of k of (C[i][k'] - u[i]).  Sources that still have excess are
      // skipped: they sit at distance 0 and act through base[] (their potential carries the lazy offset).
      for (int k = warp; k < M; k += LOSS_THREADS / 32) {
        const int cnt = s.fl_cnt[k];
        double w0 = INFINITY, w1 = INFINITY;
        int i0 = 0x7fffffff, i1 = 0x7fffffff;
        for (int q = 0; q < cnt; q += 4) {
          int ii[4], ex[4];
          double ui[4], c0[4], c1[4];
#pragma unroll
          for (int t = 0; t < 4; ++t) ii[t] = (int)s.fls[k * n + min(q + t, cnt - 1)];
#pragma unroll
          for (int t = 0; t < 4; ++t) {
            ex[t] = s.excess[ii[t]];
            ui[t] = s.u[ii[t]];
            c0[t] = has0 ? s.Cm[ii[t] * M + k0] : INFINITY;
            c1[t] = has1 ? s.Cm[ii[t] * M + k1] : INFINITY;
          }
#pragma unroll
          for (int t = 0; t < 4; ++t) {
            if (q + t < cnt && ex[t] == 0) {
              const double a0 = c0[t] - ui[t], a1 = c1[t] - ui[t];
              if (a0 < w0 || (a0 == w0 && ii[t] < i0)) { w0 = a0; i0 = ii[t]; }
              if (a1 < w1 || (a1 == w1 && ii[t] < i1)) { w1 = a1; i1 = ii[t]; }
            }
          }
        }
        // stored as arc lengths k -> k': W - v[k'] clamped at 0 (reduced costs are >= 0 up to rounding)
        s.Wv[k * OT_WLD + k0] = has0 ? fmax(w0 - s.v[k0], 0.0) : INFINITY;
        s.Wv[k * OT_WLD + k1] = has1 ? fmax(w1 - s.v[k1], 0.0) : INFINITY;
        s.Wi[k * OT_WLD + k0] = (short)(i0 == 0x7fffffff || !has0 ? -1 : i0);
        s.Wi[k * OT_WLD + k1] = (short)(i1 == 0x7fffffff || !has1 ? -1 : i1);
      }
      __syncthreads();
      if (tid < 32) {
        // ---- B: Dijkstra over the sinks (lane l owns sinks l and l + 32: distances and parents in registers).  All unsettled
        // sinks at the current minimum distance are settled in one round (arc lengths >= 0); a deficit among them ends the search.
        // (+ 0.0 turns a -0.0 into +0.0: warp_argmin orders distances by their bit patterns)
        double d0 = has0 ? fmax(s.base_v[k0] - u_ex_off - s.v[k0], 0.0) + 0.0 : INFINITY,
               d1 = has1 ? fmax(s.base_v[k1] - u_ex_off - s.v[k1], 0.0) + 0.0 : INFINITY;
        int p0_ = has0 ? s.base_i[k0] : -1, p1_ = has1 ? s.base_i[k1] : -1;   // parent source ...
        int via0 = -1, via1 = -1;                                   // ... and the sink it was reached through (-1: it has excess)
        const double v0 = has0 ? s.v[k0] : 0.0, v1 = has1 ? s.v[k1] : 0.0;
        const bool def0 = has0 && s.deficit[k0] > 0, def1 = has1 && s.deficit[k1] > 0;   // deficits do not change during a search
        bool set0 = !has0, set1 = !has1;                            // a lane's sinks past M never take part
        int target = -1, nord = 0;
        double D = 0.0;
        for (int round = 0; round <= M; ++round) {
          double bv = INFINITY;
          int bk = 0x7fffffff;
          if (!set0) { bv = d0; bk = k0; }
          if (!set1 && (d1 < bv || (d1 == bv && k1 < bk))) { bv = d1; bk = k1; }
          warp_argmin(bv, bk);
          ++n_pop;
          if (bk >= M || !(bv < INFINITY)) break;
          const bool at0 = !set0 && d0 == bv, at1 = !set1 && d1 == bv;
          const unsigned m0 = __ballot_sync(0xffffffffu, at0), m1 = __ballot_sync(0xffffffffu, at1);
          const unsigned t0 = __ballot_sync(0xffffffffu, at0 && def0);
          const unsigned t1 = __ballot_sync(0xffffffffu, at1 && def1);
          if (t0 | t1) { target = t0 ? (__ffs(t0) - 1) : (32 + __ffs(t1) - 1); D = bv; break; }
          if (at0) set0 = true;
          if (at1) set1 = true;
          // relax my unsettled sinks from the newly settled ones, in ascending sink order (minima are lexicographic in
          // (distance, parent source): the plan does not depend on lane order)
          for (int hf = 0; hf < 2; ++hf) {
            unsigned mm = hf == 0 ? m0 : m1;
            while (mm) {
              const int bit = __ffs(mm) - 1;
              mm &= mm - 1;
              const int ks = hf * 32 + bit;
              if (lane == 0) { s.ord[nord] = ks; s.dsink[nord] = bv; }
              ++nord;
              const int s0 = (int)s.Wi[ks * OT_WLD + k0], s1 = (int)s.Wi[ks * OT_WLD + k1];
              if (!set0 && s0 >= 0) {
                const double nd0 = s.Wv[ks * OT_WLD + k0] + bv;
                if (nd0 < d0 || (nd0 == d0 && s0 < p0_)) { d0 = nd0; p0_ = s0; via0 = ks; }
              }
              if (!set1 && s1 >= 0) {
                const double nd1 = s.Wv[ks * OT_WLD + k1] + bv;
                if (nd1 < d1 || (nd1 == d1 && s1 < p1_)) { d1 = nd1; p1_ = s1; via1 = ks; }
              }
            }
          }
        }
        if (target < 0) fail |= 2;
        int left = -1;                                   // a source that just lost its last unit of excess
        if (!fail) {
          if (has0 && (set0 || k0 == target)) { s.par_k[k0] = p0_; s.par_via[k0] = via0; }
          if (has1 && (set1 || k1 == target)) { s.par_k[k1] = p1_; s.par_via[k1] = via1; }
          // ---- C: potentials (kept modulo the common shift of an augmentation: u += D everywhere, v -= D everywhere leaves every
          // reduced cost unchanged).  Settled sinks: v -= D - d; a source without excess that feeds a settled sink was reached at
          // that sink's distance (the first one in settle order): u += D - d; the sources with excess share the lazy offset.
          if (has0 && set0) s.v[k0] = v0 - (D - d0);
          if (has1 && set1) s.v[k1] = v1 - (D - d1);
          __syncwarp();
          for (int o = 0; o < nord; ++o) {
            const int ks = s.ord[o];
            const double du = D - s.dsink[o];
            const int cnt = s.fl_cnt[ks];
            for (int q = lane; q < cnt; q += 32) {
              const int i = (int)s.fls[ks * n + q];
              if (s.excess[i] == 0 && s.stamp[i] != epoch) {
                s.stamp[i] = epoch;
                s.u[i] += du;
              }
            }
            __syncwarp();
          }
          u_ex_off += D;
          // ---- D: augment along the parent chain and maintain the lists (lane 0) ----
          if (lane == 0) {
            int delta = s.deficit[target];
            int k = target, i = s.par_k[k], hops = 0;
            while (s.excess[i] == 0) {                     // reached through a backward arc of sink par_via[k]
              const int pk = s.par_via[k];
              if (pk < 0 || ++hops > 2 * M + 2) { fail |= 4; delta = 0; break; }
              delta = min(delta, X(i, pk));
              k = pk;
              i = s.par_k[k];
            }
            delta = min(delta, s.excess[i]);
            if (delta > 0) {
              k = target;
              i = s.par_k[k];
              s.deficit[target] -= delta;
              while (true) {
                const int xf = X(i, k);
                if (xf == 0) s.fls[k * n + s.fl_cnt[k]++] = (short)i;      // i starts feeding k
                s.xs[i * M + k] = (signed char)(xf + delta);
                if (s.excess[i] > 0) {
                  s.excess[i] -= delta;
                  if (s.excess[i] == 0) left = i;
                  break;
                }
                const int pk = s.par_via[k];
                const int xb = X(i, pk) - delta;
                s.xs[i * M + pk] = (signed char)xb;
                if (xb == 0) {                             // i stops feeding pk: swap-remove it from pk's list
                  const int c = --s.fl_cnt[pk];
                  int q = 0;
                  while (q < c && (int)s.fls[pk * n + q] != i) ++q;
                  s.fls[pk * n + q] = s.fls[pk * n + c];
                }
                k = pk;
                i = s.par_k[k];
              }
              mass -= delta;
            } else {
              fail |= 8;
              mass = 0;
            }
          }
          mass = __shfl_sync(0xffffffffu, mass, 0);
          left = __shfl_sync(0xffffffffu, left, 0);
          fail = __shfl_sync(0xffffffffu, fail, 0);
        }
        if (!fail && left >= 0) {
          // the source leaves the excess set: materialise its potential, drop it from the list, and recompute the base of
          // the sinks whose minimiser it was (base[k] = min over the sources with excess of C_ik - u_i)
          if (lane == 0) {
            s.u[left] += u_ex_off;
            const int q = s.exq[left], last = s.exl[nex - 1];
            s.exl[q] = last;
            s.exq[last] = q;
          }
          nex -= 1;
          __syncwarp();
#pragma unroll
          for (int t = 0; t < 2; ++t) {
            const int k = t == 0 ? k0 : k1;
            if (k < M && s.base_i[k] == left) {
              double best = INFINITY;
              int bi = 0x7fffffff;
              for (int q = 0; q < nex; q += 4) {
                int ii[4];
                double cc[4];
#pragma unroll
                for (int t2 = 0; t2 < 4; ++t2) ii[t2] = s.exl[min(q + t2, nex - 1)];
#pragma unroll
                for (int t2 = 0; t2 < 4; ++t2) cc[t2] = s.Cm[ii[t2] * M + k] - s.u[ii[t2]];
#pragma unroll
                for (int t2 = 0; t2 < 4; ++t2)
                  if (q + t2 < nex && (cc[t2] < best || (cc[t2] == best && ii[t2] < bi))) { best = cc[t2]; bi = ii[t2]; }
              }
              s.base_v[k] = best;
              s.base_i[k] = bi;
            }
          }
        }
        if (lane == 0) { sh_mass = mass; sh_fail = fail; }
      }
      __syncthreads();
    }
    if (tid == 0) {
      int fail = sh_fail;
      if (sh_mass > 0) fail |= 16;
      if (fail) atomicOr(err, fail);
    }
  }
  __syncthreads();
  // ---- value and keypoint gradients from the (constant) plan T = x / (n * M) ----
  int* xg = flow + (long)p0 * M;
  const double unit = 1.0 / ((double)n * (double)M);
  double tot = 0.0;
  for (int o = tid; o < n * M; o += LOSS_THREADS) {
    const int f = (int)s.xs[o];
    xg[o] = f;                                       // publish the plan
    if (f) tot += (double)f * s.Cm[o];
  }
  tot = block_sum_d(tot, red) * unit;
  if (tid == 0) {
    parts[(long)b * 4 + 1] = tot;
    parts[(long)b * 4 + 3] = (double)n_aug + 1e-9 * (double)n_pop;     // solver statistics: augmentations + 1e-9 * search rounds
  }
  const double gsc = 2.0 * unit * w_ot / (double)B;
  for (int o = tid; o < M * 6; o += LOSS_THREADS) {
    const int k = o / 6, q = o - k * 6;
    double t = 0.0;
    for (int i = 0; i < n; ++i) {
      const int f = (int)s.xs[i * M + k];
      if (f) t += (double)f * (s.Y[k * 6 + q] - s.P[i * 6 + q]);
    }
    const int side = q / 3, c = q - side * 3;
    dkeypts[((long)(side == 0 ? b : B + b) * M + k) * 3 + c] = gsc * t;
  }
}

// loss = mean_b mse + w_ot mean_b ot + w_int mean_b inter (train.py:143-150); out[0..3] = {loss, mse, ot, inter}
__global__ void loss_total_kernel(int n_pairs, const double* __restrict__ parts, double w_ot, double w_int,
                                  double* __restrict__ out) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    double a = 0.0, b = 0.0, c = 0.0;
    for (int i = 0; i < n_pairs; ++i) { a += parts[(long)i * 4]; b += parts[(long)i * 4 + 1]; c += parts[(long)i * 4 + 2]; }
    a /= n_pairs; b /= n_pairs; c /= n_pairs;
    out[0] = a + w_ot * b + w_int * c;
    out[1] = a; out[2] = b; out[3] = c;
  }
}

}  // namespace eqd

extern "C" size_t eqd_losses_workspace_bytes_k(int32_t n_rec_nodes, int32_t n_pocket_total, int32_t n_heads) {
  const int M = eqd_valid_heads(n_heads);
  if (!M) return 0;
  const size_t a = ((size_t)(n_rec_nodes > 0 ? n_rec_nodes : 1) * 8 + 255) & ~(size_t)255;
  const size_t f = ((size_t)(n_pocket_total > 0 ? n_pocket_total : 1) * M * 4 + 255) & ~(size_t)255;
  return a + f + f / 2 + 256 + 2 * f + 256;      // flows (int32), per-sink source lists (int16), cost matrix (fp64)
}

extern "C" size_t eqd_losses_workspace_bytes(int32_t n_rec_nodes, int32_t n_pocket_total) {
  return eqd_losses_workspace_bytes_k(n_rec_nodes, n_pocket_total, EQD_HEADS);
}

extern "C" int eqd_losses(const eqd_graph* g, const float* pred_lig, const float* bound_lig, const float* bound_rec,
                          const double* keypts, const int32_t* pocket_ptr, const float* pocket_lig,
                          const float* pocket_rec, int32_t n_pocket_total, int32_t max_pocket, float w_ot, float w_int, float sigma,
                          float surface_ct, void* workspace, size_t workspace_bytes, double* parts, double* total,
                          float* dcoors, double* dkeypts, int32_t* err_flags, void* stream) {
  return eqd_losses_k(g, pred_lig, bound_lig, bound_rec, keypts, EQD_HEADS, pocket_ptr, pocket_lig, pocket_rec,
                      n_pocket_total, max_pocket, w_ot, w_int, sigma, surface_ct, workspace, workspace_bytes, parts, total,
                      dcoors, dkeypts, err_flags, stream);
}

// parts[B][4] = {mse, ot, intersection, -} per pair; total[4] = {loss, mean mse, mean ot, mean intersection};
// dcoors [N_l][3] fp32 and dkeypts [2B][K][3] fp64 = gradients of `loss`; plan_flow (inside the workspace) keeps the
// integer transport plans.  err_flags (device int, zeroed by the call) != 0 reports a pocket larger than 1024 or a solver
// failure.
extern "C" int eqd_losses_k(const eqd_graph* g, const float* pred_lig, const float* bound_lig, const float* bound_rec,
                            const double* keypts, int32_t n_heads, const int32_t* pocket_ptr, const float* pocket_lig,
                            const float* pocket_rec, int32_t n_pocket_total, int32_t max_pocket, float w_ot, float w_int,
                            float sigma, float surface_ct, void* workspace, size_t workspace_bytes, double* parts,
                            double* total, float* dcoors, double* dkeypts, int32_t* err_flags, void* stream) {
  if (!g || !pred_lig || !bound_lig || !bound_rec || !keypts || !pocket_ptr || !pocket_lig || !pocket_rec || !workspace ||
      !parts || !total || !dcoors || !dkeypts || !err_flags)
    return EQD_ERR_BAD_ARG;
  const int M = eqd_valid_heads(n_heads);
  if (!M) return EQD_ERR_UNSUPPORTED;
  const int n_rec = g->n_nodes - g->n_lig_nodes;
  if (workspace_bytes < eqd_losses_workspace_bytes_k(n_rec, n_pocket_total, M)) return EQD_ERR_WORKSPACE;
  if (g->n_pairs <= 0) return EQD_OK;
  cudaStream_t st = (cudaStream_t)stream;
  unsigned char* w = reinterpret_cast<unsigned char*>(workspace);
  double* wrec = reinterpret_cast<double*>(w);
  const size_t fbytes = ((size_t)(n_pocket_total > 0 ? n_pocket_total : 1) * M * 4 + 255) & ~(size_t)255;
  int* flow = reinterpret_cast<int*>(w + (((size_t)(n_rec > 0 ? n_rec : 1) * 8 + 255) & ~(size_t)255));
  short* lists = reinterpret_cast<short*>(reinterpret_cast<unsigned char*>(flow) + fbytes);
  double* cost = reinterpret_cast<double*>(reinterpret_cast<unsigned char*>(lists) + fbytes / 2 + 256 - ((fbytes / 2) & 255));
  cudaError_t me = cudaMemsetAsync(err_flags, 0, sizeof(int32_t), st);
  if (me != cudaSuccess) return -(1000 + (int)me);
  eqd::loss_mse_intersection_kernel<<<g->n_pairs, LOSS_THREADS, 0, st>>>(*g, pred_lig, bound_lig, bound_rec, (double)sigma,
                                                                        (double)surface_ct, (double)w_int, wrec, parts,
                                                                        dcoors);
  EQD_CUDA_LAUNCH_CHECK();
  int cap = max_pocket > 0 ? max_pocket : 1;
  if (cap > OT_MAX_POCKET) cap = OT_MAX_POCKET;            // larger pockets are flagged by the kernel (err bit 1)
  const size_t smem = eqd::ot_layout(cap, M).bytes;
  EQD_SET_SMEM((eqd::ot_emd_kernel), smem);
  eqd::ot_emd_kernel<<<g->n_pairs, LOSS_THREADS, smem, st>>>(g->n_pairs, cap, M, pocket_ptr, pocket_lig, pocket_rec, keypts,
                                                            (double)w_ot, flow, lists, cost, parts, dkeypts, err_flags);
  EQD_CUDA_LAUNCH_CHECK();
  eqd::loss_total_kernel<<<1, 32, 0, st>>>(g->n_pairs, parts, (double)w_ot, (double)w_int, total);
  EQD_CUDA_LAUNCH_CHECK();
  return EQD_OK;
}
