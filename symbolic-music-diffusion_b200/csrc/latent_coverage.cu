// Latent-space coverage metrics (sample_ncsn.py:132-159): improved precision / recall and realism (Kynkaenniemi et
// al. 2019), the PRD histograms (Sajjadi et al. 2018) and the NDB bins (Richardson & Weiss 2018), all from the Gram
// product that smd_latent_stats uses (latent_gram.cuh).  Every step after G reads G only: the squared distance of
// rows a and b is rebuilt in fp64 exactly as latent_kernel_sums_kernel does,
//   D(a, b) = max(G_aa + G_bb - 2 G_ab [+ |u - v|^2 + 2 (<c_x, u - v> - <c_y, u - v>)], 0),
// the bracket for pairs across the two sets (c_x the centred x row, u / v the mean rows).  G is made symmetric first,
// so D(a, b) = D(b, a) bit for bit.
//
// k-means runs in distance form: with S(p, C) = sum_{b in C} D(p, b) and W_C = sum_{p in C} S(p, C), the squared
// distance of p to the mean of C is S(p, C) / |C| - W_C / (2 |C|^2), and the inertia of a partition is
// sum_C W_C / (2 |C|).  One Lloyd iteration is one pass over G per fit (km_sums_kernel), then two small kernels.  All
// restarts and runs of a fit set iterate together; a per-fit converged flag on the device turns the remaining
// launches of a converged fit into no-ops, so max_iter iterations are enqueued without any host round trip and a
// converged fit costs one early-exiting block per launch.  Every reduction is in a fixed order; no atomics.
#include <climits>
#include <cmath>

#include "latent_gram.cuh"

namespace smd {

static constexpr int kCovMaxNeighbors = 32, kCovMaxClusters = 64;
static constexpr int kSeedThreads = 1024;
static constexpr int kKnnWarps = 4, kRowWarps = 8;
static constexpr int kSumWarps = 4;   // km_sums_kernel: points per block (one warp each)

struct Dist {
  const float* G;
  int Rp, n;
  const double* diag;   // [n + m] G_rr
  const double* e;      // [n + m] <c_r, u - v> = G_ru - G_rv
  const double* delta2; // |u - v|^2 from the fp64 means
  __device__ __forceinline__ double operator()(int a, int b) const {
    double s = diag[a] + diag[b] - 2.0 * static_cast<double>(G[static_cast<size_t>(a) * Rp + b]);
    if ((a < n) != (b < n)) s = s + *delta2 + 2.0 * (a < n ? e[a] - e[b] : e[b] - e[a]);
    return fmax(s, 0.0);
  }
};

// k-means state of F fits of K clusters over the points [0, N) (G rows)
struct KmFits {
  int N, K, F;
  int* labels;      // [F][N]
  double* S;        // [F][N][K] S(p, C); the seeding's min-distance scratch before the first iteration
  double* W;        // [F][K]
  int* size;        // [F][K]
  double* inertia;  // [F]
  int* state;       // [F][3]: converged, changed in the last iteration, iterations run
};

// ---- G symmetric and the per-row mean-difference terms ----------------------------------------------------------
// 32 x 32 tiles below the diagonal take the transpose of their mirror tile above it
__global__ void __launch_bounds__(1024) cov_symmetrize_kernel(float* G, int Rp, int R) {
  __shared__ float t[32][33];
  const int bi = blockIdx.y, bj = blockIdx.x;
  if (bj > bi) return;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int r = bj * 32 + ty, c = bi * 32 + tx;                 // source: upper tile (bj, bi)
  if (r < R && c < R) t[ty][tx] = G[static_cast<size_t>(r) * Rp + c];
  __syncthreads();
  const int r2 = bi * 32 + ty, c2 = bj * 32 + tx;               // destination: lower tile (bi, bj)
  if (r2 < R && c2 < R && r2 > c2) G[static_cast<size_t>(r2) * Rp + c2] = t[tx][ty];
}

__global__ void cov_e_kernel(const float* __restrict__ G, int Rp, int rows, double* __restrict__ e) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < rows)
    e[r] = static_cast<double>(G[static_cast<size_t>(rows) * Rp + r]) -
           static_cast<double>(G[static_cast<size_t>(rows + 1) * Rp + r]);
}

// ---- k-NN radii ------------------------------------------------------------------------------------------------
// One warp per row a: the k-th smallest D(a, b) over the other rows b of a's set.  Each lane keeps the k smallest of
// its strided columns sorted in shared memory; the warp then merges the 32 lists k times by value.
__global__ void __launch_bounds__(kKnnWarps * 32) cov_knn_kernel(Dist D, int n, int m, int k, double* radius) {
  __shared__ double lst[kKnnWarps][kCovMaxNeighbors][32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int a = blockIdx.x * kKnnWarps + w;
  if (a >= n + m) return;
  const int b0 = a < n ? 0 : n, b1 = a < n ? n : n + m;
  double(*L)[32] = lst[w];
  int cnt = 0;
  for (int b = b0 + lane; b < b1; b += 32) {
    if (b == a) continue;
    const double v = D(a, b);
    int pos;
    if (cnt < k) pos = cnt++;
    else if (v < L[k - 1][lane]) pos = k - 1;
    else continue;
    while (pos > 0 && L[pos - 1][lane] > v) { L[pos][lane] = L[pos - 1][lane]; --pos; }
    L[pos][lane] = v;
  }
  int head = 0;
  double r = 0.0;
  for (int i = 0; i < k; ++i) {
    double v = head < cnt ? L[head][lane] : INFINITY;
    int who = lane;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const double ov = __shfl_xor_sync(0xffffffffu, v, o);
      const int owho = __shfl_xor_sync(0xffffffffu, who, o);
      if (ov < v || (ov == v && owho < who)) { v = ov; who = owho; }
    }
    if (who == lane) ++head;
    r = v;
  }
  if (lane == 0) radius[a] = r;
}

// sorted[rank] = radius[i] for the n x radii (rank by value, then index)
__global__ void cov_rank_sort_kernel(const double* __restrict__ radius, int n, double* __restrict__ sorted) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double v = radius[i];
  int rank = 0;
  for (int j = 0; j < n; ++j) {
    const double u = radius[j];
    rank += (u < v) || (u == v && j < i);
  }
  sorted[rank] = v;
}

// One warp per row b.  flag[b]: some row a of the other set has D(a, b) <= r_a.  For b in y also realism[b - n] =
// max_a sqrt(r'_a) / (sqrt(D(a, b)) + 1e-5), r'_a = r_a, or 0 where r_a exceeds the median of the x radii
// (np.percentile(r, 50): linear interpolation between the two middle values as numpy computes it).
__global__ void __launch_bounds__(kRowWarps * 32)
cov_membership_kernel(Dist D, int n, int m, const double* __restrict__ radius, const double* __restrict__ sorted,
                      int* __restrict__ flag, double* __restrict__ realism) {
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.x * kRowWarps + (threadIdx.x >> 5);
  if (b >= n + m) return;
  const bool by = b >= n;
  const int a0 = by ? 0 : n, a1 = by ? n : n + m;
  double med = sorted[(n - 1) / 2];
  if (n % 2 == 0) {
    const double lo = sorted[n / 2 - 1], hi = sorted[n / 2];
    med = hi - (hi - lo) * 0.5;
  }
  int in = 0;
  double best = 0.0;
  for (int a = a0 + lane; a < a1; a += 32) {
    const double dd = D(b, a), r = radius[a];
    in |= dd <= r;
    if (by) best = fmax(best, sqrt(r > med ? 0.0 : r) / (sqrt(dd) + 1e-5));
  }
  in = __any_sync(0xffffffffu, in);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) best = fmax(best, __shfl_xor_sync(0xffffffffu, best, o));
  if (lane == 0) {
    flag[b] = in;
    if (by) realism[b - n] = best;
  }
}

// counts[0] = y rows inside the x manifold, counts[1] = x rows inside the y manifold
__global__ void __launch_bounds__(1024) cov_count_kernel(const int* __restrict__ flag, int n, int m, int* counts) {
  __shared__ int sx[32], sy[32];
  int cx = 0, cy = 0;
  for (int r = threadIdx.x; r < n + m; r += blockDim.x) (r < n ? cx : cy) += flag[r];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { cx += __shfl_xor_sync(0xffffffffu, cx, o); cy += __shfl_xor_sync(0xffffffffu, cy, o); }
  if ((threadIdx.x & 31) == 0) { sx[threadIdx.x >> 5] = cx; sy[threadIdx.x >> 5] = cy; }
  __syncthreads();
  if (threadIdx.x == 0) {
    int tx = 0, ty = 0;
    for (int w = 0; w < static_cast<int>(blockDim.x >> 5); ++w) { tx += sx[w]; ty += sy[w]; }
    counts[0] = ty;
    counts[1] = tx;
  }
}

// ---- k-means ---------------------------------------------------------------------------------------------------
// inclusive prefix sum over the block in thread order (fixed order); *total gets the block's sum
__device__ __forceinline__ double block_scan_f64(double v, double* red, double* total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const double u = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += u;
  }
  __syncthreads();
  if (lane == 31) red[w] = v;
  __syncthreads();
  double before = 0.0, all = 0.0;
  for (int i = 0; i < nw; ++i) {
    if (i < w) before += red[i];
    all += red[i];
  }
  *total = all;
  return before + v;
}

// k-means++ seeding of fit f (one block each) from its K uniforms, then each point to its nearest seed.  Seed 0 is
// point floor(u_0 N); seed j is the smallest index whose prefix sum (point order, fixed order) of the min squared
// distance to the seeds so far exceeds u_j times the total (floor(u_j N) if the total is 0; N - 1 if rounding leaves
// no such index).  Point p = t + 1024 i belongs to thread t.
__global__ void __launch_bounds__(kSeedThreads) km_seed_kernel(Dist D, KmFits km, const double* __restrict__ u) {
  __shared__ double red[32];
  __shared__ int found[32];
  const int f = blockIdx.x, t = threadIdx.x, N = km.N, K = km.K;
  const int rows = (N + kSeedThreads - 1) / kSeedThreads;
  const double* uf = u + static_cast<size_t>(f) * K;
  double* mind = km.S + static_cast<size_t>(f) * N * K;
  int* lab = km.labels + static_cast<size_t>(f) * N;
  int s = min(static_cast<int>(uf[0] * N), N - 1);
  for (int j = 0; j < K; ++j) {
    if (j > 0) {
      double total = 0.0, part;
      for (int i = 0; i < rows; ++i) {
        const int p = t + i * kSeedThreads;
        block_scan_f64(p < N ? mind[p] : 0.0, red, &part);
        total += part;
      }
      if (total > 0.0) {
        const double target = uf[j] * total;
        double base = 0.0;
        s = N - 1;
        for (int i = 0; i < rows; ++i) {
          const int p = t + i * kSeedThreads;
          const double pre = base + block_scan_f64(p < N ? mind[p] : 0.0, red, &part);
          base += part;
          const unsigned hit = __ballot_sync(0xffffffffu, p < N && pre > target);
          __syncthreads();
          if ((t & 31) == 0) found[t >> 5] = hit ? (t & ~31) + __ffs(hit) - 1 + i * kSeedThreads : INT_MAX;
          __syncthreads();
          int first = INT_MAX;
          for (int w = 0; w < kSeedThreads / 32; ++w) first = min(first, found[w]);
          if (first != INT_MAX) { s = first; break; }
        }
      } else {
        s = min(static_cast<int>(uf[j] * N), N - 1);
      }
    }
    for (int i = 0; i < rows; ++i) {
      const int p = t + i * kSeedThreads;
      if (p >= N) break;
      const double dd = D(s, p);
      if (j == 0 || dd < mind[p]) { mind[p] = dd; lab[p] = j; }
    }
    __syncthreads();
  }
  if (t == 0) {
    int* st = km.state + 3 * f;
    st[0] = 0; st[1] = 1; st[2] = 0;
  }
}

// start of an iteration: a fit whose last reassignment changed no label has converged
__global__ void km_check_kernel(KmFits km) {
  for (int f = blockIdx.x * blockDim.x + threadIdx.x; f < km.F; f += gridDim.x * blockDim.x) {
    int* st = km.state + 3 * f;
    if (!st[1]) st[0] = 1;
    st[1] = 0;
  }
}

// S(p, C) for every cluster C of fit f (blockIdx.y, or *fit_sel) and the points p of rows [row0, row0 + np), summed
// over the columns b in [0, N) with labels of fit f.  One warp per point; lane l adds D(p, b) for b = l (mod 32) in
// column order into its own bucket per cluster (shared memory), then the buckets are summed over the lanes in a fixed
// tree.  out rows: [F][np][K] (fit_sel: [np][K]).
__global__ void __launch_bounds__(kSumWarps * 32)
km_sums_kernel(Dist D, KmFits km, int row0, int np, const int* __restrict__ fit_sel, double* __restrict__ out) {
  extern __shared__ double bucket[];   // [kSumWarps][K][32]
  const int f = fit_sel ? *fit_sel : blockIdx.y;
  if (!fit_sel && km.state[3 * f]) return;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, K = km.K, N = km.N;
  const int i = blockIdx.x * kSumWarps + w;
  if (i >= np) return;
  const int p = row0 + i;
  double* bk = bucket + static_cast<size_t>(w) * K * 32;
  for (int c = 0; c < K; ++c) bk[c * 32 + lane] = 0.0;
  const int* lab = km.labels + static_cast<size_t>(f) * N;
  for (int b = lane; b < N; b += 32) bk[lab[b] * 32 + lane] += D(p, b);
  __syncwarp();
  double* o = out + (static_cast<size_t>(fit_sel ? 0 : f) * np + i) * K;
  for (int c = 0; c < K; ++c) {
    const double v = warp_sum_f64(bk[c * 32 + lane]);
    if (lane == 0) o[c] = v;
  }
}

// W_C = sum over the points of C (point order) of S(p, C), |C|, and the inertia sum_C W_C / (2 |C|) of fit f.
// One block per fit, one warp per cluster.
__global__ void __launch_bounds__(1024) km_within_kernel(KmFits km) {
  const int f = blockIdx.x;
  if (km.state[3 * f]) return;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, K = km.K, N = km.N;
  const int* lab = km.labels + static_cast<size_t>(f) * N;
  const double* S = km.S + static_cast<size_t>(f) * N * K;
  for (int c = w; c < K; c += blockDim.x >> 5) {
    double s = 0.0;
    int cnt = 0;
    for (int p = lane; p < N; p += 32)
      if (lab[p] == c) { s += S[static_cast<size_t>(p) * K + c]; ++cnt; }
    s = warp_sum_f64(s);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    if (lane == 0) { km.W[f * K + c] = s; km.size[f * K + c] = cnt; }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double in = 0.0;
    for (int c = 0; c < K; ++c) {
      const int cnt = km.size[f * K + c];
      if (cnt) in += km.W[f * K + c] / (2.0 * cnt);
    }
    km.inertia[f] = in;
  }
}

// argmin_C S(p, C) / |C| - W_C / (2 |C|^2) over the nonempty clusters, lowest index on ties
__device__ __forceinline__ int km_nearest(const double* S, const double* W, const int* size, int K) {
  int best = -1;
  double bd = 0.0;
  for (int c = 0; c < K; ++c) {
    const int cnt = size[c];
    if (!cnt) continue;
    const double dc = static_cast<double>(cnt);
    const double v = S[c] / dc - W[c] / (2.0 * dc * dc);
    if (best < 0 || v < bd) { best = c; bd = v; }
  }
  return best;
}

// one Lloyd reassignment of every point of every unconverged fit (thread per point)
__global__ void km_assign_kernel(KmFits km) {
  const int f = blockIdx.y;
  int* st = km.state + 3 * f;
  if (st[0]) return;
  const int p = blockIdx.x * blockDim.x + threadIdx.x, K = km.K, N = km.N;
  if (blockIdx.x == 0 && threadIdx.x == 0) ++st[2];
  if (p >= N) return;
  const int c = km_nearest(km.S + (static_cast<size_t>(f) * N + p) * K, km.W + f * K, km.size + f * K, K);
  int* lab = km.labels + static_cast<size_t>(f) * N + p;
  if (c != *lab) { *lab = c; st[1] = 1; }   // every writer stores the same 1
}

// best[r]: the restart of run r with the lowest inertia (lowest restart on ties)
__global__ void km_select_kernel(const KmFits km, int restarts, int runs, int* best, int* max_iters) {
  for (int r = threadIdx.x; r < runs; r += blockDim.x) {
    int b = 0;
    for (int i = 1; i < restarts; ++i)
      if (km.inertia[r * restarts + i] < km.inertia[r * restarts + b]) b = i;
    best[r] = b;
  }
  if (threadIdx.x == 0 && max_iters) {
    int it = 0;
    for (int f = 0; f < km.F; ++f) it = max(it, km.state[3 * f + 2]);
    *max_iters = it;
  }
}

// NDB: each y row (S rows of the best restart's clusters) to its nearest bin
__global__ void km_assign_rows_kernel(const KmFits km, const int* __restrict__ best, const double* __restrict__ S,
                                      int rows, int* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows) return;
  const int f = *best, K = km.K;
  out[i] = km_nearest(S + static_cast<size_t>(i) * K, km.W + f * K, km.size + f * K, K);
}

// hist[run][0][c] = x points of cluster c, hist[run][1][c] = y points, for the best restart of each run (one block
// per run, one thread per cluster).  PRD: labels of the union (x first); NDB: x labels, then y_labels.
__global__ void km_hist_kernel(const KmFits km, int restarts, const int* __restrict__ best, int nx, int ny,
                               const int* __restrict__ y_labels, int* __restrict__ hist) {
  const int run = blockIdx.x, c = threadIdx.x, K = km.K;
  if (c >= K) return;
  const int* lx = km.labels + static_cast<size_t>(run * restarts + best[run]) * km.N;
  const int* ly = y_labels ? y_labels : lx + nx;
  int hx = 0, hy = 0;
  for (int p = 0; p < nx; ++p) hx += lx[p] == c;
  for (int p = 0; p < ny; ++p) hy += ly[p] == c;
  hist[(run * 2) * K + c] = hx;
  hist[(run * 2 + 1) * K + c] = hy;
}

// ---- workspace ---------------------------------------------------------------------------------------------------
struct KmLayout { size_t labels, S, W, size, inertia, state, best, end; };

static KmLayout km_layout(size_t off, int N, int K, int F, int runs) {
  KmLayout L;
  L.labels = off; off = align256(off + static_cast<size_t>(F) * N * sizeof(int));
  L.S = off; off = align256(off + static_cast<size_t>(F) * N * K * sizeof(double));
  L.W = off; off = align256(off + static_cast<size_t>(F) * K * sizeof(double));
  L.size = off; off = align256(off + static_cast<size_t>(F) * K * sizeof(int));
  L.inertia = off; off = align256(off + static_cast<size_t>(F) * sizeof(double));
  L.state = off; off = align256(off + static_cast<size_t>(F) * 3 * sizeof(int));
  L.best = off; off = align256(off + static_cast<size_t>(runs) * sizeof(int));
  L.end = off;
  return L;
}

static KmFits km_fits(uint8_t* ws, const KmLayout& L, int N, int K, int F) {
  return KmFits{N, K, F, reinterpret_cast<int*>(ws + L.labels), reinterpret_cast<double*>(ws + L.S),
                reinterpret_cast<double*>(ws + L.W), reinterpret_cast<int*>(ws + L.size),
                reinterpret_cast<double*>(ws + L.inertia), reinterpret_cast<int*>(ws + L.state)};
}

struct CoverageLayout {
  GramLayout gram;
  size_t e, radius, sorted, flag, ndb_s, ndb_y;
  KmLayout prd, ndb;
  size_t total;
};

static CoverageLayout coverage_layout(int n, int m, int d, const smd_coverage_config& c) {
  CoverageLayout L;
  L.gram = gram_layout(n, m, d);
  size_t off = L.gram.total;
  L.e = off; off = align256(off + static_cast<size_t>(n + m) * sizeof(double));
  L.radius = off; off = align256(off + static_cast<size_t>(n + m) * sizeof(double));
  L.sorted = off; off = align256(off + static_cast<size_t>(n) * sizeof(double));
  L.flag = off; off = align256(off + static_cast<size_t>(n + m) * sizeof(int));
  L.ndb_s = off; off = align256(off + static_cast<size_t>(m) * c.ndb_bins * sizeof(double));
  L.ndb_y = off; off = align256(off + static_cast<size_t>(m) * sizeof(int));
  L.prd = km_layout(off, n + m, c.prd_clusters, c.prd_runs * c.restarts, c.prd_runs);
  L.ndb = km_layout(L.prd.end, n, c.ndb_bins, c.restarts, 1);
  L.total = L.ndb.end;
  return L;
}

static const char* coverage_reject(int n, int m, int d, const smd_coverage_config* c) {
  if (!c) return "null config";
  if (c->neighbors < 1 || c->neighbors > kCovMaxNeighbors) return "neighbors must be in [1, 32]";
  if (n < c->neighbors + 1 || m < c->neighbors + 1) return "both sample sets need at least neighbors + 1 rows";
  if (d < 1 || d > INT_MAX - 63) return "d must be in [1, INT_MAX - 63]";
  if (n > kLatentMaxRows - m) return "n + m must be <= 16384 (the Gram of the stacked sets)";
  if (c->prd_clusters < 1 || c->prd_clusters > kCovMaxClusters || c->prd_clusters > n + m)
    return "prd_clusters must be in [1, 64] and at most n + m";
  if (c->ndb_bins < 1 || c->ndb_bins > kCovMaxClusters || c->ndb_bins > n) return "ndb_bins must be in [1, 64] and at most n";
  if (c->restarts < 1 || c->prd_runs < 1 || c->max_iter < 1) return "restarts, prd_runs and max_iter must be >= 1";
  // labels and S of all fits are indexed with int products in places: keep F * N * K well inside size_t and the
  // grid's y extent
  if (static_cast<long long>(c->prd_runs) * c->restarts > 65535) return "prd_runs * restarts must be <= 65535";
  return nullptr;
}

// Seeds and iterates all F fits of km, then the final sums, W and inertia of the final labels.
static int run_kmeans(const Dist& D, const KmFits& km, const double* u, int max_iter, cudaStream_t st) {
  km_seed_kernel<<<km.F, kSeedThreads, 0, st>>>(D, km, u);
  CNT();
  const size_t smem = static_cast<size_t>(kSumWarps) * km.K * 32 * sizeof(double);
  SMD_CUDA(cudaFuncSetAttribute(km_sums_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  const dim3 sums_grid((km.N + kSumWarps - 1) / kSumWarps, km.F), assign_grid((km.N + 255) / 256, km.F);
  for (int it = 0; it <= max_iter; ++it) {
    km_check_kernel<<<(km.F + 255) / 256, 256, 0, st>>>(km);
    km_sums_kernel<<<sums_grid, kSumWarps * 32, smem, st>>>(D, km, 0, km.N, nullptr, km.S);
    km_within_kernel<<<km.F, 1024, 0, st>>>(km);
    CNT(); CNT(); CNT();
    if (it == max_iter) break;   // the final pass: W and inertia of the final labels
    km_assign_kernel<<<assign_grid, 256, 0, st>>>(km);
    CNT();
  }
  SMD_LAUNCH_CHECK("latent_coverage k-means");
  return SMD_OK;
}

}  // namespace smd

using namespace smd;

extern "C" {

size_t smd_latent_coverage_workspace_bytes(int n, int m, int d, const smd_coverage_config* cfg) {
  if (coverage_reject(n, m, d, cfg)) return 0;
  return coverage_layout(n, m, d, *cfg).total;
}

int smd_latent_coverage(const float* x, int n, const float* y, int m, int d, const smd_coverage_config* cfg,
                        const double* uniforms, void* workspace, size_t workspace_bytes, int* counts, double* realism,
                        int* prd_hist, int* ndb_hist, int* iterations, smd_stream_t stream) {
  if (const char* why = coverage_reject(n, m, d, cfg)) { set_error(why); return SMD_ERR_INVALID; }
  if (!x || !y || !uniforms || !workspace || !counts || !realism || !prd_hist || !ndb_hist) {
    set_error("null argument");
    return SMD_ERR_INVALID;
  }
  const smd_coverage_config c = *cfg;
  const CoverageLayout L = coverage_layout(n, m, d, c);
  if (workspace_bytes < L.total) {
    set_error("workspace too small: " + std::to_string(workspace_bytes) + " < " + std::to_string(L.total) + " bytes");
    return SMD_ERR_INVALID;
  }
  if (reinterpret_cast<uintptr_t>(workspace) & 255u) { set_error("workspace must be 256-byte aligned"); return SMD_ERR_INVALID; }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  const GramLayout& Lg = L.gram;
  if (const int rc = latent_gram(x, n, y, m, d, Lg, ws, st)) return rc;
  float* G = reinterpret_cast<float*>(ws + Lg.g);
  double* e = reinterpret_cast<double*>(ws + L.e);
  double* radius = reinterpret_cast<double*>(ws + L.radius);
  double* sorted = reinterpret_cast<double*>(ws + L.sorted);
  int* flag = reinterpret_cast<int*>(ws + L.flag);

  const int tiles = (Lg.R + 31) / 32;
  cov_symmetrize_kernel<<<dim3(tiles, tiles), 1024, 0, st>>>(G, Lg.Rp, Lg.R);
  CNT();
  cov_e_kernel<<<(n + m + 255) / 256, 256, 0, st>>>(G, Lg.Rp, n + m, e);
  CNT();
  const Dist D{G, Lg.Rp, n, reinterpret_cast<const double*>(ws + Lg.diag), e,
               reinterpret_cast<const double*>(ws + Lg.delta2)};

  // improved precision / recall and realism
  cov_knn_kernel<<<(n + m + kKnnWarps - 1) / kKnnWarps, kKnnWarps * 32, 0, st>>>(D, n, m, c.neighbors, radius);
  CNT();
  cov_rank_sort_kernel<<<(n + 255) / 256, 256, 0, st>>>(radius, n, sorted);
  CNT();
  cov_membership_kernel<<<(n + m + kRowWarps - 1) / kRowWarps, kRowWarps * 32, 0, st>>>(D, n, m, radius, sorted, flag,
                                                                                       realism);
  CNT();
  cov_count_kernel<<<1, 1024, 0, st>>>(flag, n, m, counts);
  CNT();
  SMD_LAUNCH_CHECK("latent_coverage manifolds");

  // PRD: prd_runs fits of restarts each over x and y together
  const KmFits prd = km_fits(ws, L.prd, n + m, c.prd_clusters, c.prd_runs * c.restarts);
  if (const int rc = run_kmeans(D, prd, uniforms, c.max_iter, st)) return rc;
  int* prd_best = reinterpret_cast<int*>(ws + L.prd.best);
  km_select_kernel<<<1, 256, 0, st>>>(prd, c.restarts, c.prd_runs, prd_best, iterations);
  km_hist_kernel<<<c.prd_runs, kCovMaxClusters, 0, st>>>(prd, c.restarts, prd_best, n, m, nullptr, prd_hist);
  CNT(); CNT();

  // NDB: one fit of restarts over x, then every y row to its nearest bin
  const KmFits ndb = km_fits(ws, L.ndb, n, c.ndb_bins, c.restarts);
  const double* u_ndb = uniforms + static_cast<size_t>(c.prd_runs) * c.restarts * c.prd_clusters;
  if (const int rc = run_kmeans(D, ndb, u_ndb, c.max_iter, st)) return rc;
  int* ndb_best = reinterpret_cast<int*>(ws + L.ndb.best);
  double* ndb_s = reinterpret_cast<double*>(ws + L.ndb_s);
  int* ndb_y = reinterpret_cast<int*>(ws + L.ndb_y);
  km_select_kernel<<<1, 256, 0, st>>>(ndb, c.restarts, 1, ndb_best, iterations ? iterations + 1 : nullptr);
  const size_t smem = static_cast<size_t>(kSumWarps) * ndb.K * 32 * sizeof(double);
  km_sums_kernel<<<(m + kSumWarps - 1) / kSumWarps, kSumWarps * 32, smem, st>>>(D, ndb, n, m, ndb_best, ndb_s);
  km_assign_rows_kernel<<<(m + 255) / 256, 256, 0, st>>>(ndb, ndb_best, ndb_s, m, ndb_y);
  km_hist_kernel<<<1, kCovMaxClusters, 0, st>>>(ndb, c.restarts, ndb_best, n, m, ndb_y, ndb_hist);
  CNT(); CNT(); CNT(); CNT();
  SMD_LAUNCH_CHECK("latent_coverage");
  return SMD_OK;
}

}  // extern "C"
