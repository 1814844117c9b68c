// flat_meanshift.cuh -- sklearn's flat-kernel MeanShift(bandwidth, bin_seeding=True) for one point set
// per CTA, as pvn3d/eval_icp.py:56-64 (get_cld_bigest_clus) runs it.  Shared by the segment kernel of
// flat_meanshift.cu and the ICP pre-filter of icp.cu.
//
// The steps, and the arithmetic that decides each exact output (oracle/flat_meanshift_oracle.py):
//   1. bin keys rint(x / bw) (float64 division, round-half-even); bins in order of first occurrence;
//      seed = float32(key) * float32(bw) in float32, or the points themselves when every point has its
//      own bin.
//   2. one thread per seed: members are the points with d2 <= bw*bw, d2 = (dx*dx + dy*dy) + dz*dz
//      (no FMA); no member -> stop (count 0); mean = sequential float64 sum of the members in index
//      order / count; stop when sqrt((ddx*ddx + ddy*ddy) + ddz*ddz) <= 1e-3*bw or it == max_iter.
//   3. collapse: seeds with count > 0, equal centres (==) -> the first seed's centre, the last one's count.
//   4. order by (count, x, y, z) descending (rank by counting: the keys are distinct).
//   5. greedy de-duplication in that order: a kept centre removes every later one with d2 <= bw*bw.
//   6. labels: nearest kept centre, same d2, lower index on ties.
// Every reduction runs in a fixed order, so the results are bit-identical to the oracle and run to run.
#pragma once

#include "common.cuh"

namespace pvn3d {

constexpr int kFlatMsThreads = 256;
constexpr int kFlatMsMaxPts = 4096;
// dynamic shared memory per point: the points and one more double3 (bin keys, then seed centres) as
// SoA float64, and two int arrays
constexpr size_t kFlatMsSmemPerPt = 6 * sizeof(double) + 2 * sizeof(int);

static inline size_t flat_ms_smem_bytes(int max_pts) {
  return static_cast<size_t>(max_pts < 1 ? 1 : max_pts) * kFlatMsSmemPerPt;
}

struct FlatMsOut {
  double *centres;  // [K,3] kept centres in order (may be null)
  int *counts;      // [K] member count of each kept centre (may be null)
  int *labels;      // [n] (may be null)
  int *kept;        // [n] indices of the points labelled 0, ascending (may be null)
  int *n_kept;      // [1] (may be null)
  int *n_clusters;  // [1] K (may be null)
  int *n_iter;      // [1] max completed iterations over the seeds (may be null)
};

// Shared-memory view of one fit; the caller fills x/y/z[0..n) before flat_ms_cta.
struct FlatMsSmem {
  double *x, *y, *z;     // points
  double *ax, *ay, *az;  // bin keys, then seed centres
  int *ia, *ib;
};

__device__ __forceinline__ FlatMsSmem flat_ms_smem(unsigned char *base, int cap) {
  FlatMsSmem s;
  double *d = reinterpret_cast<double *>(base);
  s.x = d;
  s.y = d + cap;
  s.z = d + 2 * cap;
  s.ax = d + 3 * cap;
  s.ay = d + 4 * cap;
  s.az = d + 5 * cap;
  s.ia = reinterpret_cast<int *>(d + 6 * cap);
  s.ib = s.ia + cap;
  return s;
}

// numpy's ((a - b)**2) summed over 3 columns: (dx*dx + dy*dy) + dz*dz, no fused multiply-add
__device__ __forceinline__ double fms_d2(double ax, double ay, double az, double bx, double by, double bz) {
  const double dx = __dsub_rn(ax, bx), dy = __dsub_rn(ay, by), dz = __dsub_rn(az, bz);
  return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}

// Exclusive scan, in index order, of flag[0..n) (0/1) into out[0..n); returns the total to every
// thread.  Each thread owns a run of consecutive elements.  flag and out may alias.
static __device__ __forceinline__ int flat_ms_scan(const int *flag, int *out, int n, int *s_warp) {
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int per = (n + kFlatMsThreads - 1) / kFlatMsThreads;
  const int c0 = min(t * per, n), c1 = min(c0 + per, n);
  int local = 0;
  for (int i = c0; i < c1; ++i) local += flag[i];
  int incl = local;
  for (int o = 1; o < 32; o <<= 1) {
    const int u = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += u;
  }
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  if (t == 0) {
    int run = 0;
    for (int w = 0; w < kFlatMsThreads / 32; ++w) {
      const int v = s_warp[w];
      s_warp[w] = run;
      run += v;
    }
    s_warp[kFlatMsThreads / 32] = run;
  }
  __syncthreads();
  int run = s_warp[warp] + incl - local;
  for (int i = c0; i < c1; ++i) {
    const int f = flag[i];
    out[i] = run;
    run += f;
  }
  const int total = s_warp[kFlatMsThreads / 32];
  __syncthreads();
  return total;
}

// One fit of n >= 1 points already in s.x/y/z.  Every thread of the CTA calls it.
static __device__ __forceinline__ void flat_ms_cta(const FlatMsSmem s, int n, double bw, int max_iter, FlatMsOut out) {
  __shared__ int s_warp[kFlatMsThreads / 32 + 1];
  __shared__ int s_iter, s_k;
  const int t = threadIdx.x;
  const double bw2 = __dmul_rn(bw, bw), thresh = __dmul_rn(1e-3, bw);
  const float bw32 = static_cast<float>(bw);
  if (t == 0) s_iter = 0;

  // 1. bin keys, first occurrences, seeds in first-occurrence order
  for (int i = t; i < n; i += kFlatMsThreads) {
    s.ax[i] = rint(__ddiv_rn(s.x[i], bw));
    s.ay[i] = rint(__ddiv_rn(s.y[i], bw));
    s.az[i] = rint(__ddiv_rn(s.z[i], bw));
  }
  __syncthreads();
  for (int i = t; i < n; i += kFlatMsThreads) {
    const double kx = s.ax[i], ky = s.ay[i], kz = s.az[i];
    int first = 1;
    for (int j = 0; j < i; ++j)
      if (s.ax[j] == kx && s.ay[j] == ky && s.az[j] == kz) {
        first = 0;
        break;
      }
    s.ia[i] = first;
  }
  __syncthreads();
  const int n_seeds = flat_ms_scan(s.ia, s.ib, n, s_warp);  // ib[i] = seed slot of point i
  int *slot_pt = reinterpret_cast<int *>(s.ax);               // the keys are no longer read
  for (int i = t; i < n; i += kFlatMsThreads)
    if (s.ia[i]) slot_pt[s.ib[i]] = i;
  __syncthreads();
  for (int sd = t; sd < n_seeds; sd += kFlatMsThreads) s.ib[sd] = slot_pt[sd];  // ib[sd] = seed's point
  __syncthreads();
  const bool seeds_are_points = n_seeds == n;

  // 2. hill climb, one thread per seed; the seed's start is recomputed from its point's key
  for (int sd = t; sd < n_seeds; sd += kFlatMsThreads) {
    const int i = s.ib[sd];
    double mx, my, mz;
    if (seeds_are_points) {
      mx = s.x[i];
      my = s.y[i];
      mz = s.z[i];
    } else {
      mx = __fmul_rn(static_cast<float>(rint(__ddiv_rn(s.x[i], bw))), bw32);
      my = __fmul_rn(static_cast<float>(rint(__ddiv_rn(s.y[i], bw))), bw32);
      mz = __fmul_rn(static_cast<float>(rint(__ddiv_rn(s.z[i], bw))), bw32);
    }
    int cnt = 0, it = 0;
    for (;;) {
      double sx = 0.0, sy = 0.0, sz = 0.0;
      int c = 0;
      for (int j = 0; j < n; ++j) {
        const double px = s.x[j], py = s.y[j], pz = s.z[j];
        if (fms_d2(px, py, pz, mx, my, mz) <= bw2) {
          sx = __dadd_rn(sx, px);
          sy = __dadd_rn(sy, py);
          sz = __dadd_rn(sz, pz);
          ++c;
        }
      }
      cnt = c;
      if (c == 0) break;
      const double fc = static_cast<double>(c);
      const double nx = __ddiv_rn(sx, fc), ny = __ddiv_rn(sy, fc), nz = __ddiv_rn(sz, fc);
      const double dx = __dsub_rn(nx, mx), dy = __dsub_rn(ny, my), dz = __dsub_rn(nz, mz);
      const double shift = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)));
      mx = nx;
      my = ny;
      mz = nz;
      if (shift <= thresh || it == max_iter) break;
      ++it;
    }
    s.ax[sd] = mx;
    s.ay[sd] = my;
    s.az[sd] = mz;
    s.ia[sd] = cnt;
    atomicMax(&s_iter, it);
  }
  __syncthreads();

  // 3. collapse equal centres: ib[sd] = the entry's count at its first seed, 0 elsewhere
  for (int sd = t; sd < n_seeds; sd += kFlatMsThreads) {
    int v = s.ia[sd];
    if (v > 0) {
      const double cx = s.ax[sd], cy = s.ay[sd], cz = s.az[sd];
      for (int j = 0; j < n_seeds; ++j) {
        if (j == sd || s.ia[j] == 0 || !(s.ax[j] == cx && s.ay[j] == cy && s.az[j] == cz)) continue;
        if (j < sd) {
          v = 0;  // not the first seed with this centre
          break;
        }
        v = s.ia[j];  // a later seed with this centre: its count wins (the last one overall)
      }
    }
    s.ib[sd] = v;
  }
  __syncthreads();

  // 4. rank of each entry under (count, x, y, z) descending; ia[rank] = seed slot
  int my_entries = 0;
  for (int sd = t; sd < n_seeds; sd += kFlatMsThreads) {
    const int c = s.ib[sd];
    if (c == 0) continue;
    ++my_entries;
    const double cx = s.ax[sd], cy = s.ay[sd], cz = s.az[sd];
    int rank = 0;
    for (int j = 0; j < n_seeds; ++j) {
      const int cj = s.ib[j];
      if (cj == 0 || j == sd) continue;
      const double xj = s.ax[j], yj = s.ay[j], zj = s.az[j];
      const bool greater =
          cj != c ? cj > c
                  : (xj != cx ? xj > cx : (yj != cy ? yj > cy : zj > cz));
      rank += greater;
    }
    s.ia[rank] = sd;
  }
  for (int o = 16; o > 0; o >>= 1) my_entries += __shfl_xor_sync(0xffffffffu, my_entries, o);
  if ((t & 31) == 0) s_warp[t >> 5] = my_entries;
  __syncthreads();
  int n_entries = 0;
  for (int w = 0; w < kFlatMsThreads / 32; ++w) n_entries += s_warp[w];
  __syncthreads();

  // 5. greedy de-duplication: a removed entry's count is negated
  for (int r = 0; r < n_entries; ++r) {
    const int sd = s.ia[r];
    if (s.ib[sd] > 0) {
      const double cx = s.ax[sd], cy = s.ay[sd], cz = s.az[sd];
      for (int q = r + 1 + t; q < n_entries; q += kFlatMsThreads) {
        const int sq = s.ia[q];
        if (s.ib[sq] > 0 && fms_d2(s.ax[sq], s.ay[sq], s.az[sq], cx, cy, cz) <= bw2) s.ib[sq] = -s.ib[sq];
      }
    }
    __syncthreads();
  }
  if (t == 0) {  // compact the kept entries in order (write index <= read index)
    int k = 0;
    for (int r = 0; r < n_entries; ++r)
      if (s.ib[s.ia[r]] > 0) s.ia[k++] = s.ia[r];
    s_k = k;
  }
  __syncthreads();
  const int K = s_k;
  for (int k = t; k < K; k += kFlatMsThreads) {
    const int sd = s.ia[k];
    if (out.centres) {
      out.centres[k * 3 + 0] = s.ax[sd];
      out.centres[k * 3 + 1] = s.ay[sd];
      out.centres[k * 3 + 2] = s.az[sd];
    }
    if (out.counts) out.counts[k] = s.ib[sd];
  }

  // 6. labels: nearest kept centre, lower index on ties (-1 when nothing was kept); ib becomes the
  // label-0 flags once every thread has passed this barrier
  __syncthreads();
  for (int i = t; i < n; i += kFlatMsThreads) {
    const double px = s.x[i], py = s.y[i], pz = s.z[i];
    int best = -1;
    double bd = 0.0;
    for (int k = 0; k < K; ++k) {
      const int sd = s.ia[k];
      const double d2 = fms_d2(px, py, pz, s.ax[sd], s.ay[sd], s.az[sd]);
      if (best < 0 || d2 < bd) {
        bd = d2;
        best = k;
      }
    }
    if (out.labels) out.labels[i] = best;
    s.ib[i] = best == 0;
  }
  __syncthreads();
  if (out.kept || out.n_kept) {
    const int nk = flat_ms_scan(s.ib, s.ia, n, s_warp);  // ia is free: the labels are written
    if (out.kept)
      for (int i = t; i < n; i += kFlatMsThreads)
        if (s.ib[i]) out.kept[s.ia[i]] = i;
    if (t == 0 && out.n_kept) *out.n_kept = nk;
  }
  if (t == 0) {
    if (out.n_clusters) *out.n_clusters = K;
    if (out.n_iter) *out.n_iter = s_iter;
  }
}

}  // namespace pvn3d
