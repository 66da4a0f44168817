// Pose Structure Score (PSS, EpipolarPose paper, Sec. 3.3): normalised 3-D poses and a
// deterministic float64 k-means (k-means++ seeding, Lloyd iterations) of the training poses.
// The reference release has no PSS code; the definition implemented here is the one in
// lib/core/pss.py and DESIGN.md section 3, and tests/pss_cases.py restates it in numpy bit
// for bit.  Every floating-point order is fixed:
//   * squared distance: sum over coordinates in index order, no FMA (--fmad=false);
//   * prefix sums, cluster sums and the inertia: points in chunks of kChunk consecutive
//     indices, each chunk summed in index order, chunk partials then added in chunk order
//     (no atomics: per-chunk partials and a fixed-order combine, as bn_bwd_partial/combine).
// CUDA cores only: the exact-distance contract rules out tensor-core dot products.
#include "common.cuh"
#include "camera.cuh"
#include <math.h>

namespace {

constexpr int kChunk = 1024;                 // points per partial
constexpr int kTile = 128;                   // points per assignment block
constexpr int kMaxSmem = 227 * 1024;         // opt-in dynamic shared memory per block (sm_90)
enum { F_CHANGED = 0, F_NONFINITE = 1, F_DUPLICATE = 2, F_COUNT = 4 };

// uniform draw j (0-based) of splitmix64 seeded by (seed, restart): top 53 bits of the output
__device__ double uniform_at(uint64_t seed, int restart, int j) {
  uint64_t z = (seed ^ ((uint64_t)restart * 0xD1B54A32D192ED03ull)) + (uint64_t)(j + 1) * 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z ^= z >> 31;
  return (double)(z >> 11) * 0x1.0p-53;
}

__host__ __device__ inline int row_pitch(int d) { return d | 1; }   // odd: conflict-free rows

// x rows [i0, i0 + kTile) -> xs[r * pitch + t]
__device__ void load_tile(const double* __restrict__ x, int64_t N, int d, int64_t i0, double* xs) {
  const int64_t n = N - i0 < kTile ? N - i0 : kTile;
  const int p = row_pitch(d);
  for (int64_t e = threadIdx.x; e < n * d; e += blockDim.x) {
    const int r = (int)(e / d), t = (int)(e - (int64_t)r * d);
    xs[r * p + t] = x[i0 * d + e];
  }
}

__device__ __forceinline__ double sqdist(const double* a, const double* c, int d) {
  double s = 0.0;
  for (int t = 0; t < d; ++t) {
    const double e = a[t] - c[t];
    s += e * e;
  }
  return s;
}

__global__ void pose_normalize_kernel(const double* __restrict__ pose, const double* __restrict__ cam,
                                      int S, int J, int root, double* __restrict__ out) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= S) return;
  const double* p = pose + (int64_t)s * J * 3;
  const double* c = cam + (int64_t)s * 5;
  double* o = out + (int64_t)s * J * 3;
  double r[3];
  cam_back_proj(p, root, c, r);
  double ss = 0.0;
  for (int j = 0; j < J; ++j) {
    double b[3];
    cam_back_proj(p, j, c, b);
    for (int k = 0; k < 3; ++k) {
      const double v = b[k] - r[k];
      o[j * 3 + k] = v;
      ss += v * v;
    }
  }
  const double nrm = sqrt(ss);
  if (nrm > 0.0)
    for (int t = 0; t < J * 3; ++t) o[t] = o[t] / nrm;
}

__global__ void nonfinite_kernel(const double* __restrict__ x, int64_t n, int32_t* flag) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    if (!isfinite(x[i])) *flag = 1;
}

// labels[i] = argmin_c |x_i - cen_c|^2 (lowest c on ties), dist2[i] = that distance;
// flag (optional) set when a label differs from the one labels[] held.
__global__ void __launch_bounds__(kTile) assign_kernel(const double* __restrict__ x, int64_t N, int d,
                                                       const double* __restrict__ cen, int k,
                                                       int32_t* __restrict__ labels, double* __restrict__ dist2,
                                                       int32_t* changed) {
  extern __shared__ double sm[];
  double* cs = sm;
  double* xs = sm + (int64_t)k * d;
  for (int e = threadIdx.x; e < k * d; e += blockDim.x) cs[e] = cen[e];
  const int64_t i0 = (int64_t)blockIdx.x * kTile;
  load_tile(x, N, d, i0, xs);
  __syncthreads();
  const int64_t i = i0 + threadIdx.x;
  if (i >= N) return;
  const double* a = xs + threadIdx.x * row_pitch(d);
  double best = INFINITY;
  int bi = 0;
  int c = 0;
  for (; c + 4 <= k; c += 4) {               // four independent sums per pass over the row
    const double* c0 = cs + (int64_t)c * d;
    double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
    for (int t = 0; t < d; ++t) {
      const double v = a[t];
      const double e0 = v - c0[t], e1 = v - c0[d + t], e2 = v - c0[2 * d + t], e3 = v - c0[3 * d + t];
      s0 += e0 * e0;
      s1 += e1 * e1;
      s2 += e2 * e2;
      s3 += e3 * e3;
    }
    if (s0 < best) { best = s0; bi = c; }
    if (s1 < best) { best = s1; bi = c + 1; }
    if (s2 < best) { best = s2; bi = c + 2; }
    if (s3 < best) { best = s3; bi = c + 3; }
  }
  for (; c < k; ++c) {
    const double s = sqdist(a, cs + (int64_t)c * d, d);
    if (s < best) { best = s; bi = c; }
  }
  if (changed && labels[i] != bi) *changed = 1;
  labels[i] = bi;
  if (dist2) dist2[i] = best;
}

// k-means++: D2[i] = min(D2[i], |x_i - cen_j|^2)   (j == 0: the distance itself)
__global__ void __launch_bounds__(kTile) kpp_dist_kernel(const double* __restrict__ x, int64_t N, int d,
                                                         const double* __restrict__ cen_j, int j,
                                                         double* __restrict__ D2) {
  extern __shared__ double sm[];
  double* cs = sm;
  double* xs = sm + d;
  for (int e = threadIdx.x; e < d; e += blockDim.x) cs[e] = cen_j[e];
  const int64_t i0 = (int64_t)blockIdx.x * kTile;
  load_tile(x, N, d, i0, xs);
  __syncthreads();
  const int64_t i = i0 + threadIdx.x;
  if (i >= N) return;
  const double s = sqdist(xs + threadIdx.x * row_pitch(d), cs, d);
  D2[i] = (j == 0 || s < D2[i]) ? s : D2[i];
}

// tot[c] = v[c*kChunk] + v[c*kChunk+1] + ... in index order (one thread per chunk)
__global__ void chunk_sum_kernel(const double* __restrict__ v, int64_t N, double* __restrict__ tot) {
  const int64_t c = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t i0 = c * kChunk;
  if (i0 >= N) return;
  const int64_t i1 = i0 + kChunk < N ? i0 + kChunk : N;
  double s = 0.0;
  for (int64_t i = i0; i < i1; ++i) s += v[i];
  tot[c] = s;
}

// out = tot[0] + tot[1] + ... in chunk order
__global__ void total_kernel(const double* __restrict__ tot, int nchunks, double* out) {
  double s = 0.0;
  for (int c = 0; c < nchunks; ++c) s += tot[c];
  *out = s;
}

// k-means++ centre j: j == 0 -> floor(u N); else the first i whose inclusive two-level prefix of
// D2 exceeds u * sum(D2) (flag F_DUPLICATE when the sum is 0).  Copies row idx to cen[j].
__global__ void kpp_select_kernel(const double* __restrict__ x, int64_t N, int d, const double* __restrict__ D2,
                                  const double* __restrict__ tot, int nchunks, uint64_t seed, int restart, int j,
                                  double* __restrict__ cen, int32_t* __restrict__ init_idx, int32_t* flags) {
  __shared__ int64_t pick;
  if (threadIdx.x == 0) {
    const double u = uniform_at(seed, restart, j);
    int64_t idx = N - 1;
    if (j == 0) {
      const int64_t f = (int64_t)(u * (double)N);
      idx = f < N - 1 ? f : N - 1;
    } else {
      double total = 0.0;
      for (int c = 0; c < nchunks; ++c) total += tot[c];
      if (total == 0.0) flags[F_DUPLICATE] = 1;
      const double target = u * total;
      double base = 0.0;
      for (int c = 0; c < nchunks; ++c) {
        const double next = base + tot[c];
        if (next > target) {
          const int64_t i0 = (int64_t)c * kChunk, i1 = i0 + kChunk < N ? i0 + kChunk : N;
          double q = 0.0;
          for (int64_t i = i0; i < i1; ++i) {
            q += D2[i];
            if (base + q > target) { idx = i; break; }
          }
          break;
        }
        base = next;
      }
    }
    pick = idx;
    init_idx[j] = (int32_t)idx;
  }
  __syncthreads();
  for (int t = threadIdx.x; t < d; t += blockDim.x) cen[(int64_t)j * d + t] = x[pick * d + t];
}

// per-chunk cluster sums (point-index order) and counts: block = chunk, thread t = coordinate t,
// thread d counts.  part [nchunks][k][d], cnt [nchunks][k].
__global__ void update_partial_kernel(const double* __restrict__ x, int64_t N, int d, int k,
                                      const int32_t* __restrict__ labels, double* __restrict__ part,
                                      int32_t* __restrict__ cnt) {
  extern __shared__ double sm[];
  double* acc = sm;                                        // [k][d]
  int32_t* n = (int32_t*)(sm + (int64_t)k * d);            // [k]
  for (int e = threadIdx.x; e < k * d; e += blockDim.x) acc[e] = 0.0;
  for (int e = threadIdx.x; e < k; e += blockDim.x) n[e] = 0;
  __syncthreads();
  const int64_t c = blockIdx.x, i0 = c * kChunk, i1 = i0 + kChunk < N ? i0 + kChunk : N;
  const int t = threadIdx.x;
  if (t < d) {
    for (int64_t i = i0; i < i1; ++i) acc[labels[i] * d + t] += x[i * d + t];
  } else if (t == d) {
    for (int64_t i = i0; i < i1; ++i) ++n[labels[i]];
  }
  __syncthreads();
  for (int e = threadIdx.x; e < k * d; e += blockDim.x) part[c * k * d + e] = acc[e];
  for (int e = threadIdx.x; e < k; e += blockDim.x) cnt[c * k + e] = n[e];
}

// cen[j][t] = (sum over chunks, in chunk order, of part[c][j][t]) / count_j for count_j > 0
__global__ void update_combine_kernel(const double* __restrict__ part, const int32_t* __restrict__ cnt,
                                      int nchunks, int d, int k, double* __restrict__ cen,
                                      int32_t* __restrict__ count) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= k * d) return;
  const int j = e / d;
  int64_t m = 0;
  for (int c = 0; c < nchunks; ++c) m += cnt[(int64_t)c * k + j];
  double s = 0.0;
  for (int c = 0; c < nchunks; ++c) s += part[(int64_t)c * k * d + e];
  if (m > 0) cen[e] = s / (double)m;
  if (e - j * d == 0) count[j] = (int32_t)m;
}

// Empty clusters, in increasing cluster order, take the points in decreasing order of dist2
// (ties: lower index first); each point at most once.  One block.
__global__ void __launch_bounds__(1024) relocate_kernel(const double* __restrict__ x, int64_t N, int d, int k,
                                                        const int32_t* __restrict__ count,
                                                        const double* __restrict__ dist2, double* __restrict__ cen) {
  __shared__ double wd[32];
  __shared__ int64_t wi[32];
  __shared__ int64_t pick;
  double pd = INFINITY;                      // the previous pick: (pd, pi) in the order
  int64_t pi = -1;
  for (int j = 0; j < k; ++j) {
    if (count[j] != 0) continue;
    double bd = -1.0;
    int64_t bi = -1;
    for (int64_t i = threadIdx.x; i < N; i += blockDim.x) {
      const double v = dist2[i];
      if (!(v < pd || (v == pd && i > pi))) continue;        // taken already
      if (v > bd || (v == bd && (bi < 0 || i < bi))) { bd = v; bi = i; }
    }
    for (int o = 16; o > 0; o >>= 1) {
      const double od = __shfl_xor_sync(0xffffffffu, bd, o);
      const int64_t oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (oi >= 0 && (bi < 0 || od > bd || (od == bd && oi < bi))) { bd = od; bi = oi; }
    }
    if ((threadIdx.x & 31) == 0) { wd[threadIdx.x >> 5] = bd; wi[threadIdx.x >> 5] = bi; }
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int w = 1; w < (int)(blockDim.x >> 5); ++w)
        if (wi[w] >= 0 && (bi < 0 || wd[w] > bd || (wd[w] == bd && wi[w] < bi))) { bd = wd[w]; bi = wi[w]; }
      pick = bi;
      wd[0] = bd;
    }
    __syncthreads();
    const int64_t p = pick;
    const double v = wd[0];
    __syncthreads();
    if (p < 0) break;                         // every point taken (k > N cannot reach here)
    for (int t = threadIdx.x; t < d; t += blockDim.x) cen[(int64_t)j * d + t] = x[p * d + t];
    pd = v;
    pi = p;
  }
}

struct KmWs {
  double* dist2;      // [N]
  double* tot;        // [nchunks]
  double* part;       // [nchunks][k][d]
  int32_t* cnt;       // [nchunks][k]
  int32_t* count;     // [k]
  int32_t* flags;     // [F_COUNT]
  double* scalar;     // [1]
};

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

size_t km_layout(int64_t N, int d, int k, char* base, KmWs* w) {
  const int64_t nch = (N + kChunk - 1) / kChunk;
  const size_t sz[7] = {align256(N * 8), align256(nch * 8), align256(nch * k * d * 8), align256(nch * k * 4),
                        align256((size_t)k * 4), align256(F_COUNT * 4), align256(8)};
  size_t off[7], o = 0;
  for (int i = 0; i < 7; ++i) { off[i] = o; o += sz[i]; }
  if (w) {
    w->dist2 = (double*)(base + off[0]);
    w->tot = (double*)(base + off[1]);
    w->part = (double*)(base + off[2]);
    w->cnt = (int32_t*)(base + off[3]);
    w->count = (int32_t*)(base + off[4]);
    w->flags = (int32_t*)(base + off[5]);
    w->scalar = (double*)(base + off[6]);
  }
  return o;
}

size_t assign_smem(int d, int k) { return ((size_t)k * d + (size_t)kTile * row_pitch(d)) * 8; }
size_t update_smem(int d, int k) { return (size_t)k * d * 8 + (size_t)k * 4; }

int check_shapes(int64_t N, int d, int k) {
  EPB_CHECK_ARG(N >= 1 && d >= 1 && k >= 1);
  if (k > N) {
    epb_set_error("k-means: k = %d exceeds the number of points N = %lld", k, (long long)N);
    return EPB_EINVAL;
  }
  if (assign_smem(d, k) > (size_t)kMaxSmem || d + 1 > 1024) {
    epb_set_error("k-means: k = %d, d = %d needs %zu bytes of shared memory (limit %d)", k, d,
                  assign_smem(d, k), kMaxSmem);
    return EPB_EINVAL;
  }
  return EPB_OK;
}

int launch_assign(const double* x, int64_t N, int d, const double* cen, int k, int32_t* labels, double* dist2,
                  int32_t* changed, cudaStream_t st) {
  const size_t smem = assign_smem(d, k);
  EPB_CUDA(cudaFuncSetAttribute(assign_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  assign_kernel<<<(unsigned)((N + kTile - 1) / kTile), kTile, smem, st>>>(x, N, d, cen, k, labels, dist2, changed);
  EPB_LAUNCH_CHECK();
  return EPB_OK;
}

int read_flag(const int32_t* dev, int32_t* host, cudaStream_t st) {
  EPB_CUDA(cudaMemcpyAsync(host, dev, sizeof(int32_t) * F_COUNT, cudaMemcpyDeviceToHost, st));
  EPB_CUDA(cudaStreamSynchronize(st));
  return EPB_OK;
}

}  // namespace

extern "C" __attribute__((visibility("default"))) int epb_pose_normalize(
    const double* pose, const double* cam, int S, int J, int root, double* out, epb_stream_t stream) {
  EPB_CHECK_ARG(pose && cam && out);
  EPB_CHECK_ARG(S >= 0 && J > 0 && root >= 0 && root < J);
  if (S == 0) return EPB_OK;
  pose_normalize_kernel<<<(S + 127) / 128, 128, 0, as_stream(stream)>>>(pose, cam, S, J, root, out);
  EPB_LAUNCH_CHECK();
  return EPB_OK;
}

extern "C" __attribute__((visibility("default"))) int epb_kmeans_workspace(int N, int d, int k, int64_t* ws_bytes) {
  EPB_CHECK_ARG(ws_bytes);
  const int rc = check_shapes(N, d, k);
  if (rc != EPB_OK) return rc;
  *ws_bytes = (int64_t)km_layout(N, d, k, nullptr, nullptr);
  return EPB_OK;
}

extern "C" __attribute__((visibility("default"))) int epb_kmeans_assign(
    const double* x, int N, int d, const double* centroids, int k, int32_t* labels, double* dist2,
    epb_stream_t stream) {
  EPB_CHECK_ARG(x && centroids && labels);
  EPB_CHECK_ARG(N >= 0 && d >= 1 && k >= 1);
  if (assign_smem(d, k) > (size_t)kMaxSmem) {
    epb_set_error("k-means: k = %d, d = %d needs %zu bytes of shared memory (limit %d)", k, d, assign_smem(d, k),
                  kMaxSmem);
    return EPB_EINVAL;
  }
  if (N == 0) return EPB_OK;
  cudaStream_t st = as_stream(stream);
  int32_t* flags = nullptr;
  int rc = epb_workspace(EPB_WS_KMEANS, sizeof(int32_t) * F_COUNT, st, (void**)&flags);
  if (rc != EPB_OK) return rc;
  EPB_CUDA(cudaMemsetAsync(flags, 0, sizeof(int32_t) * F_COUNT, st));
  nonfinite_kernel<<<256, 256, 0, st>>>(x, (int64_t)N * d, flags + F_NONFINITE);
  nonfinite_kernel<<<4, 256, 0, st>>>(centroids, (int64_t)k * d, flags + F_NONFINITE);
  EPB_LAUNCH_CHECK();
  int32_t h[F_COUNT];
  if ((rc = read_flag(flags, h, st)) != EPB_OK) return rc;
  if (h[F_NONFINITE]) {
    epb_set_error("k-means assign: non-finite point or centroid");
    return EPB_EINVAL;
  }
  return launch_assign(x, N, d, centroids, k, labels, dist2, nullptr, st);
}

extern "C" __attribute__((visibility("default"))) int epb_kmeans_fit(
    const double* x, int N, int d, int k, uint64_t seed, int restart, int max_iter, double* centroids,
    int32_t* labels, int32_t* init_idx, int32_t* trace, void* ws, int64_t ws_bytes, double* inertia_host,
    int32_t* n_iter_host, epb_stream_t stream) {
  EPB_CHECK_ARG(x && centroids && labels && init_idx && ws && inertia_host && n_iter_host);
  EPB_CHECK_ARG(max_iter >= 0 && restart >= 0);
  int rc = check_shapes(N, d, k);
  if (rc != EPB_OK) return rc;
  KmWs w;
  const size_t need = km_layout(N, d, k, (char*)ws, &w);
  if ((size_t)ws_bytes < need) {
    epb_set_error("k-means: workspace of %lld bytes, %zu needed", (long long)ws_bytes, need);
    return EPB_EINVAL;
  }
  cudaStream_t st = as_stream(stream);
  const int nch = (int)((N + kChunk - 1) / kChunk);
  const unsigned tiles = (unsigned)((N + kTile - 1) / kTile);
  EPB_CUDA(cudaMemsetAsync(w.flags, 0, sizeof(int32_t) * F_COUNT, st));
  nonfinite_kernel<<<256, 256, 0, st>>>(x, (int64_t)N * d, w.flags + F_NONFINITE);
  // k-means++ seeding
  const size_t kpp_smem = ((size_t)d + (size_t)kTile * row_pitch(d)) * 8;
  EPB_CUDA(cudaFuncSetAttribute(kpp_dist_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kpp_smem));
  for (int j = 0; j < k; ++j) {
    kpp_select_kernel<<<1, 64, 0, st>>>(x, N, d, w.dist2, w.tot, nch, seed, restart, j, centroids, init_idx,
                                        w.flags);
    if (j + 1 == k) break;
    kpp_dist_kernel<<<tiles, kTile, kpp_smem, st>>>(x, N, d, centroids + (int64_t)j * d, j, w.dist2);
    chunk_sum_kernel<<<(nch + 127) / 128, 128, 0, st>>>(w.dist2, N, w.tot);
  }
  EPB_LAUNCH_CHECK();
  int32_t h[F_COUNT];
  if ((rc = read_flag(w.flags, h, st)) != EPB_OK) return rc;
  if (h[F_NONFINITE]) {
    epb_set_error("k-means: non-finite input");
    return EPB_EINVAL;
  }
  if (h[F_DUPLICATE]) {
    epb_set_error("k-means: fewer than k = %d distinct points", k);
    return EPB_EINVAL;
  }
  // Lloyd: assignment pass 0, then (update, assignment) until no label changes or max_iter updates
  if ((rc = launch_assign(x, N, d, centroids, k, labels, w.dist2, nullptr, st)) != EPB_OK) return rc;
  if (trace) EPB_CUDA(cudaMemcpyAsync(trace, labels, (size_t)N * 4, cudaMemcpyDeviceToDevice, st));
  const size_t usmem = update_smem(d, k);
  EPB_CUDA(cudaFuncSetAttribute(update_partial_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)usmem));
  const int uthreads = (d + 1 + 31) / 32 * 32;
  int it = 0;
  while (it < max_iter) {
    update_partial_kernel<<<nch, uthreads, usmem, st>>>(x, N, d, k, labels, w.part, w.cnt);
    update_combine_kernel<<<(k * d + 127) / 128, 128, 0, st>>>(w.part, w.cnt, nch, d, k, centroids, w.count);
    relocate_kernel<<<1, 1024, 0, st>>>(x, N, d, k, w.count, w.dist2, centroids);
    EPB_CUDA(cudaMemsetAsync(w.flags + F_CHANGED, 0, sizeof(int32_t), st));
    if ((rc = launch_assign(x, N, d, centroids, k, labels, w.dist2, w.flags + F_CHANGED, st)) != EPB_OK) return rc;
    ++it;
    if (trace)
      EPB_CUDA(cudaMemcpyAsync(trace + (int64_t)it * N, labels, (size_t)N * 4, cudaMemcpyDeviceToDevice, st));
    if ((rc = read_flag(w.flags, h, st)) != EPB_OK) return rc;
    if (!h[F_CHANGED]) break;
  }
  chunk_sum_kernel<<<(nch + 127) / 128, 128, 0, st>>>(w.dist2, N, w.tot);
  total_kernel<<<1, 1, 0, st>>>(w.tot, nch, w.scalar);
  EPB_LAUNCH_CHECK();
  EPB_CUDA(cudaMemcpyAsync(inertia_host, w.scalar, sizeof(double), cudaMemcpyDeviceToHost, st));
  EPB_CUDA(cudaStreamSynchronize(st));
  *n_iter_host = it;
  return EPB_OK;
}
