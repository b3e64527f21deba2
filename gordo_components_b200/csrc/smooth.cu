// K6: optional smoothing of the anomaly columns (reference diff.py:302-308, 387-415):
//   smm  = rolling(window).median()   sma = rolling(window).mean()   (first window-1 rows NaN, pandas min_periods=window:
//                                                                     a window holding a NaN gives NaN)
//   ewma = ewm(span=window).mean()    (pandas defaults adjust=True, ignore_na=False, min_periods=0: NaNs add no observation
//                                      but age the weights, the previous average is carried forward; leading NaNs stay NaN)
// Rolling windows of different rows are independent, so smm / sma run as (column, row-chunk) work items: a thread rebuilds the
// window state at the start of its chunk (sorted window: insertion of window-1 values; mean: a sum) and then slides it over
// CHUNK rows -- O(window) per row for the median, with thousands of threads in flight instead of one per column.  Lanes run
// along columns, so every step of a warp reads one contiguous row segment.  Sums are double (pandas computes in float64).
// ewma is a recurrence over all earlier rows and stays one thread per column (a handful of flops per row).
#include <math_constants.h>
#include "gb_common.cuh"

namespace {

constexpr int SM_THREADS = 64;
constexpr int SM_CHUNK = 128;  // rows per work item of the rolling kernels

// One column of one job, rows [t0, t1) (the rolling methods) or all of them (ewma): src / dst point at the job's first row of the
// column, element t at src[t * stride].  The kernels below only decide which column a thread owns; gb_smooth and gb_smooth_scores
// share these bodies, so a column comes out with the same bits from either.  In is float or double; a double is rounded to float
// as it is read, exactly the float32 array the host would have passed.
template <typename In>
__device__ __forceinline__ float load_f32(const In* p) { return (float)*p; }

template <typename In>
__device__ __forceinline__ void sma_column(const In* src, long stride, float* dst, long dstride, int t0, int t1, int window) {
  double sum = 0.0;
  int bad = 0;  // NaNs currently inside the window
  for (int t = max(0, t0 - window); t < t0; ++t) {  // window state as the row before the chunk left it: rows [t0 - window, t0)
    const float v = load_f32(src + t * stride);
    if (v == v) sum += (double)v; else ++bad;
  }
  for (int t = t0; t < t1; ++t) {
    const float v = load_f32(src + t * stride);
    if (v == v) sum += (double)v; else ++bad;
    if (t >= window) {
      const float old = load_f32(src + (t - window) * stride);
      if (old == old) sum -= (double)old; else --bad;
    }
    dst[t * dstride] = (t >= window - 1 && bad == 0) ? (float)(sum / (double)window) : CUDART_NAN_F;
  }
}

// pandas/_libs/window/aggregations.pyx ewm() [3P, pandas 1.5.3 pinned by the reference], adjust=True, ignore_na=False, minp=1
template <typename In>
__device__ __forceinline__ void ewma_column(const In* src, long stride, float* dst, long dstride, int n_rows, int window) {
  const double alpha = 2.0 / ((double)window + 1.0), old_wt_factor = 1.0 - alpha, new_wt = 1.0;
  double weighted = (double)load_f32(src), old_wt = 1.0;
  dst[0] = (float)weighted;  // NaN when the first value is NaN
  for (int t = 1; t < n_rows; ++t) {
    const double cur = (double)load_f32(src + t * stride);
    const bool is_obs = cur == cur;
    if (weighted == weighted) {
      old_wt *= old_wt_factor;  // ignore_na=False: a missing value still ages the weights
      if (is_obs) {
        if (weighted != cur) weighted = (old_wt * weighted + new_wt * cur) / (old_wt + new_wt);
        old_wt += new_wt;
      }
    } else if (is_obs) {
      weighted = cur;
    }
    dst[t * dstride] = (float)weighted;
  }
}

// rolling median: sorted window of the non-NaN values, element i at win[i * nthr] (a [window][nthreads] shared array, so the lanes
// of a warp hit different banks)
template <typename In>
__device__ __forceinline__ void median_column(const In* src, long stride, float* dst, long dstride, int t0, int t1, int window, float* win,
                                              int nthr) {
  int count = 0, bad = 0;  // sorted values held / NaNs currently inside the window
  auto insert = [&](float v) {
    if (!(v == v)) { ++bad; return; }
    int pos = count;
    while (pos > 0 && win[(pos - 1) * nthr] > v) {
      win[pos * nthr] = win[(pos - 1) * nthr];
      --pos;
    }
    win[pos * nthr] = v;
    ++count;
  };
  auto remove = [&](float old) {
    if (!(old == old)) { --bad; return; }
    int lo = 0, hi = count;  // first element not below `old` (it is present)
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (win[mid * nthr] < old) lo = mid + 1; else hi = mid;
    }
    for (int i = lo; i + 1 < count; ++i) win[i * nthr] = win[(i + 1) * nthr];
    --count;
  };
  for (int t = max(0, t0 - window); t < t0; ++t) insert(load_f32(src + t * stride));  // window state as the row before the chunk left it
  for (int t = t0; t < t1; ++t) {
    if (t >= window) remove(load_f32(src + (t - window) * stride));
    insert(load_f32(src + t * stride));
    float m = CUDART_NAN_F;
    if (t >= window - 1 && bad == 0) {  // count == window
      const int h = window >> 1;
      m = (window & 1) ? win[h * nthr] : 0.5f * (win[(h - 1) * nthr] + win[h * nthr]);
    }
    dst[t * dstride] = m;
  }
}

__global__ void __launch_bounds__(SM_THREADS) smooth_sma_kernel(const gb_job* jobs, int job0, const float* arr, int n_cols, int window, float* out) {
  const gb_job job = jobs[job0 + blockIdx.y];
  const int j = blockIdx.x * SM_THREADS + threadIdx.x;
  const int t0 = blockIdx.z * SM_CHUNK;
  if (j >= n_cols || t0 >= job.n_rows) return;
  sma_column(arr + job.out_row * (long)n_cols + j, n_cols, out + job.out_row * (long)n_cols + j, n_cols, t0, min(job.n_rows, t0 + SM_CHUNK),
             window);
}

__global__ void __launch_bounds__(SM_THREADS) smooth_ewma_kernel(const gb_job* jobs, int job0, const float* arr, int n_cols, int window, float* out) {
  const gb_job job = jobs[job0 + blockIdx.y];
  const int j = blockIdx.x * SM_THREADS + threadIdx.x;
  if (j >= n_cols || job.n_rows <= 0) return;
  ewma_column(arr + job.out_row * (long)n_cols + j, n_cols, out + job.out_row * (long)n_cols + j, n_cols, job.n_rows, window);
}

__global__ void __launch_bounds__(SM_THREADS) smooth_median_kernel(const gb_job* jobs, int job0, const float* arr, int n_cols, int window, float* out) {
  extern __shared__ float s_win[];
  const gb_job job = jobs[job0 + blockIdx.y];
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  const int t0 = blockIdx.z * SM_CHUNK;
  if (j >= n_cols || t0 >= job.n_rows) return;
  median_column(arr + job.out_row * (long)n_cols + j, n_cols, out + job.out_row * (long)n_cols + j, n_cols, t0, min(job.n_rows, t0 + SM_CHUNK),
                window, s_win + threadIdx.x, (int)blockDim.x);
}

// The four anomaly arrays of a batch as one grid of 2T + 2 columns: [0, T) the columns of tag-anomaly-scaled, [T, 2T) those of
// tag-anomaly-unscaled, 2T total-anomaly-scaled, 2T + 1 total-anomaly-unscaled.  A thread finds its array and stride and runs the
// same column body gb_smooth runs, so the per-row arrays fill lanes of the tag arrays' CTAs instead of CTAs of their own.
struct ScoreArrays {
  const void* in[4];  // tag scaled, total scaled, tag unscaled, total unscaled
  float* out[4];
};

template <typename In>
__device__ __forceinline__ bool score_column(const ScoreArrays& a, int c, int T, const gb_job& job, const In*& src, float*& dst, long& stride) {
  if (c >= 2 * T + 2) return false;
  // selects, not a[i] with a runtime i: an indexed kernel parameter would be copied to local memory first
  const bool tag = c < 2 * T, scaled = tag ? c < T : c == 2 * T;
  const void* in = tag ? (scaled ? a.in[0] : a.in[2]) : (scaled ? a.in[1] : a.in[3]);
  float* out = tag ? (scaled ? a.out[0] : a.out[2]) : (scaled ? a.out[1] : a.out[3]);
  stride = tag ? T : 1;
  const long ofs = job.out_row * stride + (tag ? (scaled ? c : c - T) : 0);
  src = static_cast<const In*>(in) + ofs;
  dst = out + ofs;
  return true;
}

template <typename In, int METHOD>
__global__ void __launch_bounds__(SM_THREADS) smooth_scores_kernel(const gb_job* jobs, int job0, ScoreArrays a, int T, int window) {
  extern __shared__ float s_win[];
  const gb_job job = jobs[job0 + blockIdx.y];
  const int t0 = blockIdx.z * SM_CHUNK;
  const In* src;
  float* dst;
  long stride;
  if (t0 >= job.n_rows || !score_column<In>(a, blockIdx.x * blockDim.x + threadIdx.x, T, job, src, dst, stride)) return;
  const int t1 = min(job.n_rows, t0 + SM_CHUNK);
  if (METHOD == 0) median_column(src, stride, dst, stride, t0, t1, window, s_win + threadIdx.x, (int)blockDim.x);
  else if (METHOD == 1) sma_column(src, stride, dst, stride, t0, t1, window);
  else ewma_column(src, stride, dst, stride, job.n_rows, window);
}

// x'[r][c] = x[r][c] * a[slot][c] + b[slot][c] in double, rounded once to float: what sklearn's per-feature scalers compute
// in float64 before Keras casts the batch to floatx.
__global__ void affine_f64_kernel(const gb_job* __restrict__ jobs, const double* __restrict__ x, int n_cols, const double* __restrict__ a,
                                  const double* __restrict__ b, float* __restrict__ out, int job0) {
  const gb_job job = jobs[job0 + blockIdx.y];
  const long total = (long)job.n_rows * n_cols;
  const double* src = x + (long)job.x_row * n_cols;
  float* dst = out + (long)job.out_row * n_cols;
  const double* ja = a + (long)job.slot * n_cols;
  const double* jb = b + (long)job.slot * n_cols;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % n_cols);
    dst[i] = (float)(__dmul_rn(src[i], ja[c]) + jb[c]);  // two roundings like numpy's X *= scale; X += min (no fma contraction)
  }
}

// q-quantile of the non-NaN values of one column of one job (pandas Series.quantile, interpolation="linear").
// Fast path (the column fits in shared memory): compacted, padded with +inf to a power of two, bitonic sort, linear
// interpolation at (n-1)*q.
constexpr int Q_THREADS = 1024;
__device__ __forceinline__ float quantile_interp(float vlo, float vhi, double frac) {
  return (float)((double)vlo + ((double)vhi - (double)vlo) * frac);
}
__global__ void __launch_bounds__(Q_THREADS) quantile_kernel(const gb_job* __restrict__ jobs, int job0, const float* __restrict__ arr, int n_cols, float q,
                                                             float* __restrict__ out) {
  extern __shared__ float sv[];
  __shared__ int s_n;
  const gb_job job = jobs[job0 + blockIdx.y];
  const int col = blockIdx.x, tid = threadIdx.x;
  const float* src = arr + (long)job.out_row * n_cols + col;
  if (tid == 0) s_n = 0;
  __syncthreads();
  for (int r = tid; r < job.n_rows; r += Q_THREADS) {
    const float v = src[(long)r * n_cols];
    if (v == v) sv[atomicAdd(&s_n, 1)] = v;  // order is irrelevant before a sort
  }
  __syncthreads();
  const int n = s_n;
  int p2 = 1;
  while (p2 < n) p2 <<= 1;
  for (int i = n + tid; i < p2; i += Q_THREADS) sv[i] = __int_as_float(0x7f800000);
  __syncthreads();
  for (int k = 2; k <= p2; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < p2; i += Q_THREADS) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const float a = sv[i], b = sv[ixj];
          const bool up = (i & k) == 0;
          if ((a > b) == up) { sv[i] = b; sv[ixj] = a; }
        }
      }
      __syncthreads();
    }
  if (tid == 0) {
    float res = __int_as_float(0x7fc00000);  // all-NaN / empty column -> NaN, as pandas
    if (n > 0) {
      const double pos = (double)(n - 1) * (double)q;
      const int lo = (int)floor(pos), hi = min(lo + 1, n - 1);
      res = quantile_interp(sv[lo], sv[hi], pos - (double)lo);
    }
    out[(long)(job0 + blockIdx.y) * n_cols + col] = res;
  }
}

// General path (any number of rows, no workspace): the two order statistics are found by selection instead of sorting.  Floats
// map monotonically to unsigned keys; the r-th smallest key is the largest K with count(key < K) <= r, built bit by bit from the
// top (32 counting passes over the column, which stays in L2), then one pass yields count(key <= K) and the next larger key.
__device__ __forceinline__ unsigned fkey(float v) {
  const unsigned b = __float_as_uint(v);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float fkey_inv(unsigned k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

__global__ void __launch_bounds__(Q_THREADS) quantile_select_kernel(const gb_job* __restrict__ jobs, int job0, const float* __restrict__ arr, int n_cols,
                                                                    float q, float* __restrict__ out) {
  __shared__ unsigned s_cnt[2];
  __shared__ unsigned s_min;
  const gb_job job = jobs[job0 + blockIdx.y];
  const int col = blockIdx.x, tid = threadIdx.x;
  const float* src = arr + (long)job.out_row * n_cols + col;
  auto count_below = [&](unsigned bound, bool inclusive) -> unsigned {  // block-wide count of keys < bound (<= if inclusive); NaNs never count
    __syncthreads();
    if (tid == 0) s_cnt[0] = 0;
    __syncthreads();
    unsigned c = 0;
    for (int r = tid; r < job.n_rows; r += Q_THREADS) {
      const float v = __ldg(src + (long)r * n_cols);
      if (v == v) {
        const unsigned k = fkey(v);
        c += inclusive ? (k <= bound) : (k < bound);
      }
    }
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if ((tid & 31) == 0 && c) atomicAdd(&s_cnt[0], c);
    __syncthreads();
    return s_cnt[0];
  };
  const unsigned n = count_below(0xffffffffu, true);
  if (n == 0) {
    if (tid == 0) out[(long)(job0 + blockIdx.y) * n_cols + col] = __int_as_float(0x7fc00000);
    return;
  }
  const double pos = (double)(n - 1) * (double)q;
  const unsigned r = (unsigned)floor(pos);
  unsigned K = 0;
  for (int bit = 31; bit >= 0; --bit) {
    const unsigned cand = K | (1u << bit);
    if (count_below(cand, false) <= r) K = cand;
  }
  const unsigned le = count_below(K, true);
  float vhi = fkey_inv(K);
  if (le < r + 2 && r + 1 < n) {  // the next order statistic is the smallest key above K
    __syncthreads();
    if (tid == 0) s_min = 0xffffffffu;
    __syncthreads();
    unsigned m = 0xffffffffu;
    for (int rr = tid; rr < job.n_rows; rr += Q_THREADS) {
      const float v = __ldg(src + (long)rr * n_cols);
      if (v == v) {
        const unsigned k = fkey(v);
        if (k > K) m = min(m, k);
      }
    }
    for (int o = 16; o > 0; o >>= 1) m = min(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((tid & 31) == 0) atomicMin(&s_min, m);
    __syncthreads();
    vhi = fkey_inv(s_min);
  }
  if (tid == 0) out[(long)(job0 + blockIdx.y) * n_cols + col] = quantile_interp(fkey_inv(K), vhi, pos - (double)r);
}

constexpr int MAX_GRID_Y = 65535;  // gridDim.y carries the job index: larger fleets go out as several launches (job0 = first job)

}  // namespace


extern "C" int gb_quantile(const gb_job* jobs, int32_t n_jobs, int32_t max_rows, const float* arr, int32_t n_cols, float q, float* out,
                           void* stream) {
  GB_REQUIRE(jobs && arr && out, GB_E_ARG, "jobs/arr/out must be non-NULL");
  GB_REQUIRE(n_cols >= 1 && n_cols <= 65535 && max_rows >= 0, GB_E_ARG, "n_cols=%d max_rows=%d", n_cols, max_rows);
  GB_REQUIRE(q >= 0.f && q <= 1.f, GB_E_ARG, "percentiles should all be in the interval [0, 1], got %g", (double)q);
  GB_REQUIRE(n_jobs >= 0, GB_E_ARG, "bad n_jobs");
  if (n_jobs == 0) return GB_OK;
  int cap = 1;
  while (cap < max_rows) cap <<= 1;
  const size_t smem = (size_t)cap * sizeof(float);
  const bool fits = smem <= 128 * 1024;  // up to 32768 rows per job sort in shared memory; longer jobs select from L2
  if (fits) GB_CUDA_CHECK(cudaFuncSetAttribute(quantile_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  for (int j0 = 0; j0 < n_jobs; j0 += MAX_GRID_Y) {
    const dim3 grid(n_cols, n_jobs - j0 < MAX_GRID_Y ? n_jobs - j0 : MAX_GRID_Y);
    if (fits) quantile_kernel<<<grid, Q_THREADS, smem, (cudaStream_t)stream>>>(jobs, j0, arr, n_cols, q, out);
    else quantile_select_kernel<<<grid, Q_THREADS, 0, (cudaStream_t)stream>>>(jobs, j0, arr, n_cols, q, out);
  }
  GB_CUDA_CHECK(cudaGetLastError());
  return GB_OK;
}

extern "C" int gb_affine_f64(const gb_job* jobs, int32_t n_jobs, int32_t max_rows, const double* x, int32_t n_cols, const double* a,
                             const double* b, float* out, void* stream) {
  GB_REQUIRE(jobs && x && a && b && out, GB_E_ARG, "jobs/x/a/b/out must be non-NULL");
  GB_REQUIRE(n_cols >= 1 && max_rows >= 0, GB_E_ARG, "n_cols=%d max_rows=%d", n_cols, max_rows);
  GB_REQUIRE(n_jobs >= 0, GB_E_ARG, "bad n_jobs");
  if (n_jobs == 0 || max_rows == 0) return GB_OK;
  const long per_job = (long)max_rows * n_cols;
  const int bx = (int)((per_job + 256L * 8 - 1) / (256L * 8));
  for (int j0 = 0; j0 < n_jobs; j0 += MAX_GRID_Y) {
    const dim3 grid(bx < 1 ? 1 : (bx > 1184 ? 1184 : bx), n_jobs - j0 < MAX_GRID_Y ? n_jobs - j0 : MAX_GRID_Y);
    affine_f64_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(jobs, x, n_cols, a, b, out, j0);
  }
  GB_CUDA_CHECK(cudaGetLastError());
  return GB_OK;
}

namespace {

// Threads per CTA of the rolling median and the shared memory they need: one sorted window per thread, so wide windows run
// fewer columns per CTA.  false when even one thread's window does not fit.
constexpr size_t MEDIAN_SMEM_MAX = 200 * 1024;
bool median_block(int window, int& nthr, size_t& smem) {
  nthr = SM_THREADS;
  while (nthr > 1 && (size_t)window * nthr * sizeof(float) > MEDIAN_SMEM_MAX) nthr >>= 1;
  smem = (size_t)window * nthr * sizeof(float);
  return smem <= MEDIAN_SMEM_MAX;
}

template <typename In>
int launch_smooth_scores(const gb_job* jobs, int n_jobs, int max_rows, const ScoreArrays& a, int T, int window, int method, cudaStream_t st) {
  const int chunks = (max_rows + SM_CHUNK - 1) / SM_CHUNK;
  const int n_cols = 2 * T + 2;
  int nthr = SM_THREADS;
  size_t smem = 0;
  if (method == 0) {
    median_block(window, nthr, smem);
    GB_CUDA_CHECK(cudaFuncSetAttribute(smooth_scores_kernel<In, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  }
  for (int j0 = 0; j0 < n_jobs; j0 += MAX_GRID_Y) {
    const int nj = n_jobs - j0 < MAX_GRID_Y ? n_jobs - j0 : MAX_GRID_Y;
    if (method == 0) smooth_scores_kernel<In, 0><<<dim3((n_cols + nthr - 1) / nthr, nj, chunks), nthr, smem, st>>>(jobs, j0, a, T, window);
    else if (method == 1) smooth_scores_kernel<In, 1><<<dim3((n_cols + SM_THREADS - 1) / SM_THREADS, nj, chunks), SM_THREADS, 0, st>>>(jobs, j0, a, T, window);
    else smooth_scores_kernel<In, 2><<<dim3((n_cols + SM_THREADS - 1) / SM_THREADS, nj), SM_THREADS, 0, st>>>(jobs, j0, a, T, window);
  }
  GB_CUDA_CHECK(cudaGetLastError());
  return GB_OK;
}

}  // namespace

extern "C" int gb_smooth(const gb_job* jobs, int32_t n_jobs, int32_t max_rows, const float* arr, int32_t n_cols, int32_t window, int32_t method,
                         float* out, void* stream) {
  GB_REQUIRE(jobs && arr && out, GB_E_ARG, "jobs/arr/out must be non-NULL");
  GB_REQUIRE(n_cols >= 1 && window >= 1, GB_E_ARG, "n_cols=%d window=%d must be >= 1", n_cols, window);
  GB_REQUIRE(method >= 0 && method <= 2, GB_E_ARG, "method=%d unknown (0 smm, 1 sma, 2 ewma)", method);
  GB_REQUIRE(n_jobs >= 0 && max_rows >= 0, GB_E_ARG, "bad n_jobs / max_rows");
  if (n_jobs == 0 || max_rows == 0) return GB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int chunks = (max_rows + SM_CHUNK - 1) / SM_CHUNK;
  GB_REQUIRE(chunks <= 65535, GB_E_ARG, "smoothing handles at most %d rows per job", 65535 * SM_CHUNK);
  int nthr = SM_THREADS;
  size_t smem = 0;
  if (method == 0) {
    GB_REQUIRE(median_block(window, nthr, smem), GB_E_SMEM, "rolling-median window %d exceeds the %d values one thread's sorted window may hold",
               window, (int)(MEDIAN_SMEM_MAX / sizeof(float)));
    GB_CUDA_CHECK(cudaFuncSetAttribute(smooth_median_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  }
  for (int j0 = 0; j0 < n_jobs; j0 += MAX_GRID_Y) {
    const int nj = n_jobs - j0 < MAX_GRID_Y ? n_jobs - j0 : MAX_GRID_Y;
    if (method == 0) smooth_median_kernel<<<dim3((n_cols + nthr - 1) / nthr, nj, chunks), nthr, smem, st>>>(jobs, j0, arr, n_cols, window, out);
    else if (method == 1) smooth_sma_kernel<<<dim3((n_cols + SM_THREADS - 1) / SM_THREADS, nj, chunks), SM_THREADS, 0, st>>>(jobs, j0, arr, n_cols, window, out);
    else smooth_ewma_kernel<<<dim3((n_cols + SM_THREADS - 1) / SM_THREADS, nj), SM_THREADS, 0, st>>>(jobs, j0, arr, n_cols, window, out);
  }
  GB_CUDA_CHECK(cudaGetLastError());
  return GB_OK;
}

extern "C" int gb_smooth_scores(const gb_job* jobs, int32_t n_jobs, int32_t max_rows, const void* tag_scaled, const void* total_scaled,
                                const void* tag_unscaled, const void* total_unscaled, int32_t in_f64, int32_t n_tags, int32_t window, int32_t method,
                                float* smooth_tag_scaled, float* smooth_total_scaled, float* smooth_tag_unscaled, float* smooth_total_unscaled,
                                void* stream) {
  GB_REQUIRE(jobs && tag_scaled && total_scaled && tag_unscaled && total_unscaled, GB_E_ARG, "jobs and the four score arrays must be non-NULL");
  GB_REQUIRE(smooth_tag_scaled && smooth_total_scaled && smooth_tag_unscaled && smooth_total_unscaled, GB_E_ARG,
             "the four smoothed outputs must be non-NULL");
  GB_REQUIRE(in_f64 == 0 || in_f64 == 1, GB_E_ARG, "in_f64=%d must be 0 (float32 scores) or 1 (float64)", in_f64);
  GB_REQUIRE(n_tags >= 1 && n_tags <= (1 << 24), GB_E_ARG, "n_tags=%d must be in [1, %d]", n_tags, 1 << 24);
  GB_REQUIRE(window >= 1, GB_E_ARG, "window=%d must be >= 1", window);
  GB_REQUIRE(method >= 0 && method <= 2, GB_E_ARG, "method=%d unknown (0 smm, 1 sma, 2 ewma)", method);
  GB_REQUIRE(n_jobs >= 0 && max_rows >= 0, GB_E_ARG, "bad n_jobs / max_rows");
  GB_REQUIRE((max_rows + SM_CHUNK - 1) / SM_CHUNK <= 65535, GB_E_ARG, "smoothing handles at most %d rows per job", 65535 * SM_CHUNK);
  int nthr;
  size_t smem;
  GB_REQUIRE(method != 0 || median_block(window, nthr, smem), GB_E_SMEM,
             "rolling-median window %d exceeds the %d values one thread's sorted window may hold", window, (int)(MEDIAN_SMEM_MAX / sizeof(float)));
  if (n_jobs == 0 || max_rows == 0) return GB_OK;
  const ScoreArrays a{{tag_scaled, total_scaled, tag_unscaled, total_unscaled},
                      {smooth_tag_scaled, smooth_total_scaled, smooth_tag_unscaled, smooth_total_unscaled}};
  cudaStream_t st = (cudaStream_t)stream;
  return in_f64 ? launch_smooth_scores<double>(jobs, n_jobs, max_rows, a, n_tags, window, method, st)
                : launch_smooth_scores<float>(jobs, n_jobs, max_rows, a, n_tags, window, method, st);
}
