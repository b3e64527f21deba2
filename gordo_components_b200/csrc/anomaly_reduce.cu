// K5 + K7: the two small column reductions of the anomaly path, and the scoring of existing predictions.
//   gb_minmax_fit : sklearn MinMaxScaler.fit on the targets (reference diff.py:173)
//   gb_thresholds : rolling(window).min().max() per tag and for the aggregate series (diff.py:222-233)
//   gb_anomaly_score[_f64], gb_minmax_inverse_score_f64 : the anomaly columns of a prediction, the latter after the
//                   TransformedTargetRegressor's MinMax inverse in the same pass
// Both are HBM-bound single passes over [rows][n_out] arrays: lanes run along the tag axis so every warp
// request is one contiguous segment, partial results meet in shared memory and one atomic per (CTA, column)
// publishes them.
#include <math_constants.h>
#include "gb_common.cuh"
#include "postprocess.cuh"

namespace {

constexpr int THREADS = 256;
constexpr int NWARPS = THREADS / 32;
constexpr int ROWS_PER_CTA = 1024;

// The integer form follows the sign bit, not v >= 0: -0.0 is INT_MIN as a signed integer and must take the unsigned path
// of the negative values, where it is the largest.
__device__ __forceinline__ void atomic_max_float(float* addr, float v) {
  if (!signbit(v)) atomicMax(reinterpret_cast<int*>(addr), __float_as_int(v));
  else atomicMin(reinterpret_cast<unsigned*>(addr), __float_as_uint(v));
}
__device__ __forceinline__ void atomic_min_float(float* addr, float v) {
  if (!signbit(v)) atomicMin(reinterpret_cast<int*>(addr), __float_as_int(v));
  else atomicMax(reinterpret_cast<unsigned*>(addr), __float_as_uint(v));
}

// per-type constants and the integer view used by the atomic min / max below
template <typename T> struct RollBits;
template <> struct RollBits<float> {
  using I = int;
  static __device__ __forceinline__ I bits(float v) { return __float_as_int(v); }
  static __device__ __forceinline__ float nan() { return CUDART_NAN_F; }
  static __device__ __forceinline__ float inf() { return CUDART_INF_F; }
};
template <> struct RollBits<double> {
  using I = long long;
  static __device__ __forceinline__ I bits(double v) { return __double_as_longlong(v); }
  static __device__ __forceinline__ double nan() { return CUDART_NAN; }
  static __device__ __forceinline__ double inf() { return CUDART_INF; }
};

// ---------------------------------------------------------------- min / max per column
// IEEE values of one sign order like (or against) their bit patterns: a float / double min or max is an integer atomic.
__device__ __forceinline__ void atomic_max_fp(float* addr, float v) { atomic_max_float(addr, v); }
__device__ __forceinline__ void atomic_min_fp(float* addr, float v) { atomic_min_float(addr, v); }
__device__ __forceinline__ void atomic_max_fp(double* addr, double v) {
  if (!signbit(v)) atomicMax(reinterpret_cast<long long*>(addr), __double_as_longlong(v));
  else atomicMin(reinterpret_cast<unsigned long long*>(addr), (unsigned long long)__double_as_longlong(v));
}
__device__ __forceinline__ void atomic_min_fp(double* addr, double v) {
  if (!signbit(v)) atomicMin(reinterpret_cast<long long*>(addr), __double_as_longlong(v));
  else atomicMax(reinterpret_cast<unsigned long long*>(addr), (unsigned long long)__double_as_longlong(v));
}

template <typename T>
__global__ void minmax_init_kernel(const gb_job* jobs, int n_out, T* ws) {
  const gb_job job = jobs[blockIdx.x];
  T* w = ws + (long)job.slot * 2 * n_out;
  for (int j = threadIdx.x; j < n_out; j += blockDim.x) {
    w[j] = RollBits<T>::inf();            // running min
    w[n_out + j] = -RollBits<T>::inf();   // running max
  }
}

template <typename T>
__global__ void __launch_bounds__(THREADS) minmax_reduce_kernel(const gb_job* jobs, int job0, const T* y, int n_out, T* ws) {
  __shared__ T s_min[NWARPS][GB_MAX_WIDTH];
  __shared__ T s_max[NWARPS][GB_MAX_WIDTH];
  const gb_job job = jobs[job0 + blockIdx.y];
  const int r0 = blockIdx.x * ROWS_PER_CTA;
  if (r0 >= job.n_rows) return;
  const int r1 = min(job.n_rows, r0 + ROWS_PER_CTA);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const T* base = y + job.x_row * (long)n_out;
  for (int j0 = 0; j0 < n_out; j0 += 32) {
    const int j = j0 + lane;
    T lo = RollBits<T>::inf(), hi = -RollBits<T>::inf();
    if (j < n_out) {
      for (int r = r0 + warp; r < r1; r += NWARPS) {
        const T v = __ldg(base + (long)r * n_out + j);
        if (v == v) { lo = v < lo ? v : lo; hi = v > hi ? v : hi; }   // NaNs are skipped (sklearn uses nanmin / nanmax)
      }
      s_min[warp][j] = lo;
      s_max[warp][j] = hi;
    }
  }
  __syncthreads();
  T* w = ws + (long)job.slot * 2 * n_out;
  for (int j = threadIdx.x; j < n_out; j += THREADS) {
    T lo = s_min[0][j], hi = s_max[0][j];
#pragma unroll
    for (int q = 1; q < NWARPS; ++q) { lo = s_min[q][j] < lo ? s_min[q][j] : lo; hi = s_max[q][j] > hi ? s_max[q][j] : hi; }
    if (lo <= hi) {  // at least one finite sample
      atomic_min_fp(&w[j], lo);
      atomic_max_fp(&w[n_out + j], hi);
    }
  }
}

__global__ void minmax_finalize_kernel(const gb_job* jobs, int n_out, const float* ws, float* scale, float* offset) {
  const gb_job job = jobs[blockIdx.x];
  const float* w = ws + (long)job.slot * 2 * n_out;
  for (int j = threadIdx.x; j < n_out; j += blockDim.x) {
    const float lo = w[j], hi = w[n_out + j];
    float range = hi - lo;
    // sklearn _handle_zeros_in_scale: ranges below 10*eps are treated as 1 (constant feature)
    if (!(range >= 10.f * 1.1920929e-7f)) range = 1.f;
    const float s = 1.f / range;
    scale[(long)job.slot * n_out + j] = s;
    if (offset) offset[(long)job.slot * n_out + j] = -lo * s;
  }
}

// ---------------------------------------------------------------- rolling(window).min().max() per column
// T = float for the scores of this package's fp32 networks, double for the float64 arithmetic the reference applies to
// foreign base estimators (diff.py:268-300 on float64 y).  Non-negative IEEE values order like their bit patterns, so the
// running maximum is an integer atomicMax; -1 marks "no complete window yet".
template <typename T>
__global__ void rollmax_init_kernel(const gb_job* jobs, int n_cols, T* out) {
  const gb_job job = jobs[blockIdx.x];
  for (int j = threadIdx.x; j < n_cols; j += blockDim.x) out[(long)job.slot * n_cols + j] = (T)-1;
}

// arr: [rows][n_cols] (non-negative values); positions t in [window-1, n_rows) of each job.
template <typename T>
__global__ void __launch_bounds__(THREADS) rollmin_max_kernel(const gb_job* jobs, int job0, const T* arr, int n_cols, int window,
                                                               T* out) {
  __shared__ T s_max[NWARPS][GB_MAX_WIDTH];
  const gb_job job = jobs[job0 + blockIdx.y];
  const int t0 = window - 1 + blockIdx.x * ROWS_PER_CTA;
  if (t0 >= job.n_rows) return;
  const int t1 = min(job.n_rows, t0 + ROWS_PER_CTA);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const T* base = arr + job.out_row * (long)n_cols;
  for (int j0 = 0; j0 < n_cols; j0 += 32) {
    const int j = j0 + lane;
    if (j < n_cols) {
      T best = (T)-1;
      for (int t = t0 + warp; t < t1; t += NWARPS) {
        T m = RollBits<T>::inf();
        bool nan = false;
        for (int i = 0; i < window; ++i) {
          const T v = __ldg(base + (long)(t - i) * n_cols + j);
          nan |= !(v == v);
          m = v < m ? v : m;
        }
        if (!nan) best = m > best ? m : best;  // pandas: a window holding NaN yields NaN, which max() skips
      }
      s_max[warp][j] = best;
    }
  }
  __syncthreads();
  for (int j = threadIdx.x; j < n_cols; j += THREADS) {
    T best = s_max[0][j];
#pragma unroll
    for (int q = 1; q < NWARPS; ++q) best = s_max[q][j] > best ? s_max[q][j] : best;
    best = best + (T)0;  // -0.0 -> +0.0: as an integer -0.0 would never beat the -1 marker
    if (best >= (T)0)
      atomicMax(reinterpret_cast<typename RollBits<T>::I*>(&out[(long)job.slot * n_cols + j]), RollBits<T>::bits(best));
  }
}

template <typename T>
__global__ void rollmax_finalize_kernel(const gb_job* jobs, int n_cols, T* out) {
  const gb_job job = jobs[blockIdx.x];
  for (int j = threadIdx.x; j < n_cols; j += blockDim.x) {
    T* p = &out[(long)job.slot * n_cols + j];
    if (*p < (T)0) *p = RollBits<T>::nan();  // fewer rows than the window: pandas gives NaN
  }
}

// ---------------------------------------------------------------- score of existing predictions (diff.py:350-385, 420-444)
// T = float: predictions of this package's fp32 networks; T = double: the reference's float64 arithmetic
// (diff.py:268-300, 350-385 run pandas on float64 y) for predictions that did not come from an fp32 network here.
template <typename T>
__global__ void __launch_bounds__(THREADS) anomaly_score_kernel(const gb_job* jobs, int job0, const T* yhat, const T* y, int n_out,
                                                                 const T* scale, const T* feat_thr,
                                                                 const T* agg_thr, T* o_ts, T* o_tu,
                                                                 T* o_tots, T* o_totu, T* o_conf,
                                                                 T* o_totconf) {
  const gb_job job = jobs[job0 + blockIdx.y];
  const int r0 = blockIdx.x * ROWS_PER_CTA;
  if (r0 >= job.n_rows) return;
  const int r1 = min(job.n_rows, r0 + ROWS_PER_CTA);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const T* sc = scale ? scale + (long)job.slot * n_out : nullptr;
  const T* ft = feat_thr ? feat_thr + (long)job.slot * n_out : nullptr;
  const T inv = (T)1 / (T)n_out;
  for (int r = r0 + warp; r < r1; r += NWARPS) {
    const long go = (job.out_row + r) * (long)n_out, gy = (job.x_row + r) * (long)n_out;
    GB_SCORE_ROW(T, __ldg(yhat + go + j));
  }
}

// The TransformedTargetRegressor's prediction scored in one pass: every element of the network's float32 output p goes through
// the slot's MinMax inverse (y_scale / y_min), is stored to out_model and is scored as a double against the float64 y, exactly
// as minmax_inverse_kernel followed by anomaly_score_kernel<double> on its widened output compute it.  p and out_model may be
// the same array (each element is read before the same thread overwrites it), so neither goes through the read-only path.
__global__ void __launch_bounds__(THREADS) minmax_inverse_score_kernel(const gb_job* jobs, int job0, const float* p, const double* y, int n_out,
                                                                        const double* y_scale, const double* y_min,
                                                                        const double* scale, const double* feat_thr,
                                                                        const double* agg_thr, float* out_model, double* o_ts,
                                                                        double* o_tu, double* o_tots, double* o_totu,
                                                                        double* o_conf, double* o_totconf) {
  const gb_job job = jobs[job0 + blockIdx.y];
  const int r0 = blockIdx.x * ROWS_PER_CTA;
  if (r0 >= job.n_rows) return;
  const int r1 = min(job.n_rows, r0 + ROWS_PER_CTA);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const double* sc = scale ? scale + (long)job.slot * n_out : nullptr;
  const double* ft = feat_thr ? feat_thr + (long)job.slot * n_out : nullptr;
  const double* ys = y_scale + (long)job.slot * n_out;
  const double* ym = y_min + (long)job.slot * n_out;
  const double inv = 1.0 / (double)n_out;
  for (int r = r0 + warp; r < r1; r += NWARPS) {
    const long go = (job.out_row + r) * (long)n_out, gy = (job.x_row + r) * (long)n_out;
    const auto yhat = [&](int j) {
      const float v = gb_post::minmax_inverse(p[go + j], ym + j, ys + j);
      out_model[go + j] = v;
      return (double)v;
    };
    GB_SCORE_ROW(double, yhat(j));
  }
}

// ---------------------------------------------------------------- column moments of one CV fold (build_model.py:378-446)
// The builder's cross-validation metrics (explained variance, r2, MSE, MAE: per tag and averaged) are all functions of five
// per-column sums over the fold's test rows.  out[job][q][j] (double), with e = yhat - y and y0 = the job's first target row
// (a shift that keeps the second moment of y well conditioned):  q=0 sum e, 1 sum e^2, 2 sum |e|, 3 sum (y-y0), 4 sum (y-y0)^2.
// One CTA per job and a fixed summation order: the result does not depend on the launch.
__global__ void __launch_bounds__(THREADS) cv_moments_kernel(const gb_job* jobs, const float* yhat, const float* y, int n_out,
                                                              double* out) {
  __shared__ double s_acc[NWARPS][5][32];
  const gb_job job = jobs[blockIdx.x];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float* yb = y + job.x_row * (long)n_out;
  const float* pb = yhat + job.out_row * (long)n_out;
  double* o = out + (long)blockIdx.x * 5 * n_out;
  for (int j0 = 0; j0 < n_out; j0 += 32) {
    const int j = j0 + lane;
    double a0 = 0., a1 = 0., a2 = 0., a3 = 0., a4 = 0.;
    if (j < n_out && job.n_rows > 0) {
      const double y0 = (double)__ldg(yb + j);
      for (int r = warp; r < job.n_rows; r += NWARPS) {
        const double yv = (double)__ldg(yb + (long)r * n_out + j);
        const double e = (double)__ldg(pb + (long)r * n_out + j) - yv;
        const double c = yv - y0;
        a0 += e; a1 += e * e; a2 += fabs(e); a3 += c; a4 += c * c;
      }
    }
    s_acc[warp][0][lane] = a0; s_acc[warp][1][lane] = a1; s_acc[warp][2][lane] = a2; s_acc[warp][3][lane] = a3; s_acc[warp][4][lane] = a4;
    __syncthreads();
    if (threadIdx.x < 5 * 32) {
      const int q = threadIdx.x >> 5;
      if (j < n_out) {
        double t = s_acc[0][q][lane];
#pragma unroll
        for (int w = 1; w < NWARPS; ++w) t += s_acc[w][q][lane];
        o[q * n_out + j] = t;
      }
    }
    __syncthreads();
  }
}

// gridDim.y carries the job index and is limited to 65535: larger fleets go out as several launches (job0 = first job).
constexpr int MAX_GRID_Y = 65535;

template <typename T>
int anomaly_score_launch(const gb_job* jobs, int32_t n_jobs, int32_t max_rows, const T* yhat, const T* y, int32_t n_out,
                         const T* scale, const T* feat_thr, const T* agg_thr, T* out_tag_scaled, T* out_tag_unscaled,
                         T* out_total_scaled, T* out_total_unscaled, T* out_conf, T* out_total_conf, void* stream) {
  GB_REQUIRE(jobs && yhat && y, GB_E_ARG, "jobs/yhat/y must be non-NULL");
  GB_REQUIRE(n_out >= 1, GB_E_SHAPE, "n_out=%d must be >= 1", n_out);
  GB_REQUIRE(scale || (!out_tag_scaled && !out_total_scaled && !out_total_conf), GB_E_ARG, "scaled outputs requested without scale");
  GB_REQUIRE(!out_conf || feat_thr, GB_E_ARG, "out_conf requested without feat_thr");
  GB_REQUIRE(!out_total_conf || agg_thr, GB_E_ARG, "out_total_conf requested without agg_thr");
  GB_REQUIRE(n_jobs >= 0, GB_E_ARG, "bad n_jobs");
  if (n_jobs == 0 || max_rows <= 0) return GB_OK;
  const int chunks = (max_rows + ROWS_PER_CTA - 1) / ROWS_PER_CTA;
  for (int j0 = 0; j0 < n_jobs; j0 += MAX_GRID_Y)
    anomaly_score_kernel<T><<<dim3(chunks, min(MAX_GRID_Y, n_jobs - j0)), THREADS, 0, (cudaStream_t)stream>>>(
        jobs, j0, yhat, y, n_out, scale, feat_thr, agg_thr, out_tag_scaled, out_tag_unscaled, out_total_scaled,
        out_total_unscaled, out_conf, out_total_conf);
  GB_CUDA_CHECK(cudaGetLastError());
  return GB_OK;
}

template <typename T>
int thresholds_launch(const gb_job* jobs, int32_t n_jobs, int32_t max_rows, const T* tag_unscaled, const T* total_scaled,
                      int32_t n_out, int32_t window, T* feat_thr, T* agg_thr, int32_t n_slots, void* stream) {
  GB_REQUIRE(jobs, GB_E_ARG, "jobs must be non-NULL");
  GB_REQUIRE((tag_unscaled != nullptr) == (feat_thr != nullptr), GB_E_ARG, "tag_unscaled and feat_thr go together");
  GB_REQUIRE((total_scaled != nullptr) == (agg_thr != nullptr), GB_E_ARG, "total_scaled and agg_thr go together");
  GB_REQUIRE(n_out >= 1 && n_out <= GB_MAX_WIDTH, GB_E_SHAPE, "n_out=%d outside [1,%d]", n_out, GB_MAX_WIDTH);
  GB_REQUIRE(window >= 1, GB_E_ARG, "window=%d must be >= 1", window);
  GB_REQUIRE(n_jobs >= 0 && n_slots >= 0, GB_E_ARG, "bad n_jobs/n_slots");
  if (n_jobs == 0) return GB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int span = max_rows - (window - 1);
  const int chunks = span > 0 ? (span + ROWS_PER_CTA - 1) / ROWS_PER_CTA : 0;
  if (feat_thr) {
    rollmax_init_kernel<T><<<n_jobs, 128, 0, st>>>(jobs, n_out, feat_thr);
    for (int j0 = 0; chunks && j0 < n_jobs; j0 += MAX_GRID_Y)
      rollmin_max_kernel<T><<<dim3(chunks, min(MAX_GRID_Y, n_jobs - j0)), THREADS, 0, st>>>(jobs, j0, tag_unscaled, n_out, window, feat_thr);
    rollmax_finalize_kernel<T><<<n_jobs, 128, 0, st>>>(jobs, n_out, feat_thr);
  }
  if (agg_thr) {
    rollmax_init_kernel<T><<<n_jobs, 32, 0, st>>>(jobs, 1, agg_thr);
    for (int j0 = 0; chunks && j0 < n_jobs; j0 += MAX_GRID_Y)
      rollmin_max_kernel<T><<<dim3(chunks, min(MAX_GRID_Y, n_jobs - j0)), THREADS, 0, st>>>(jobs, j0, total_scaled, 1, window, agg_thr);
    rollmax_finalize_kernel<T><<<n_jobs, 32, 0, st>>>(jobs, 1, agg_thr);
  }
  GB_CUDA_CHECK(cudaGetLastError());
  return GB_OK;
}

}  // namespace

extern "C" {

int gb_anomaly_score(const gb_job* jobs, int32_t n_jobs, int32_t max_rows, const float* yhat, const float* y,
                     int32_t n_out, const float* scale, const float* feat_thr, const float* agg_thr,
                     float* out_tag_scaled, float* out_tag_unscaled, float* out_total_scaled,
                     float* out_total_unscaled, float* out_conf, float* out_total_conf, void* stream) {
  return anomaly_score_launch<float>(jobs, n_jobs, max_rows, yhat, y, n_out, scale, feat_thr, agg_thr, out_tag_scaled,
                                     out_tag_unscaled, out_total_scaled, out_total_unscaled, out_conf, out_total_conf, stream);
}

int gb_anomaly_score_f64(const gb_job* jobs, int32_t n_jobs, int32_t max_rows, const double* yhat, const double* y,
                         int32_t n_out, const double* scale, const double* feat_thr, const double* agg_thr,
                         double* out_tag_scaled, double* out_tag_unscaled, double* out_total_scaled,
                         double* out_total_unscaled, double* out_conf, double* out_total_conf, void* stream) {
  return anomaly_score_launch<double>(jobs, n_jobs, max_rows, yhat, y, n_out, scale, feat_thr, agg_thr, out_tag_scaled,
                                      out_tag_unscaled, out_total_scaled, out_total_unscaled, out_conf, out_total_conf, stream);
}

int gb_minmax_inverse_score_f64(const gb_job* jobs, int32_t n_jobs, int32_t max_rows, const float* p, const double* y,
                                int32_t n_out, const double* y_scale, const double* y_min, const double* scale,
                                const double* feat_thr, const double* agg_thr, float* out_model,
                                double* out_tag_scaled, double* out_tag_unscaled, double* out_total_scaled,
                                double* out_total_unscaled, double* out_conf, double* out_total_conf, void* stream) {
  GB_REQUIRE(jobs && p && y && y_scale && y_min && out_model, GB_E_ARG, "jobs/p/y/y_scale/y_min/out_model must be non-NULL");
  GB_REQUIRE(n_out >= 1, GB_E_SHAPE, "n_out=%d must be >= 1", n_out);
  GB_REQUIRE(scale || (!out_tag_scaled && !out_total_scaled && !out_total_conf), GB_E_ARG, "scaled outputs requested without scale");
  GB_REQUIRE(!out_conf || feat_thr, GB_E_ARG, "out_conf requested without feat_thr");
  GB_REQUIRE(!out_total_conf || agg_thr, GB_E_ARG, "out_total_conf requested without agg_thr");
  GB_REQUIRE(n_jobs >= 0, GB_E_ARG, "bad n_jobs");
  if (n_jobs == 0 || max_rows <= 0) return GB_OK;
  const int chunks = (max_rows + ROWS_PER_CTA - 1) / ROWS_PER_CTA;
  for (int j0 = 0; j0 < n_jobs; j0 += MAX_GRID_Y)
    minmax_inverse_score_kernel<<<dim3(chunks, min(MAX_GRID_Y, n_jobs - j0)), THREADS, 0, (cudaStream_t)stream>>>(
        jobs, j0, p, y, n_out, y_scale, y_min, scale, feat_thr, agg_thr, out_model, out_tag_scaled, out_tag_unscaled, out_total_scaled,
        out_total_unscaled, out_conf, out_total_conf);
  GB_CUDA_CHECK(cudaGetLastError());
  return GB_OK;
}

int gb_minmax_fit(const gb_job* jobs, int32_t n_jobs, int32_t max_rows, const float* y, int32_t n_out, float* scale,
                  float* offset, float* minmax_ws, int32_t n_slots, void* stream) {
  GB_REQUIRE(jobs && y && scale && minmax_ws, GB_E_ARG, "jobs/y/scale/minmax_ws must be non-NULL");
  GB_REQUIRE(n_out >= 1 && n_out <= GB_MAX_WIDTH, GB_E_SHAPE, "n_out=%d outside [1,%d]", n_out, GB_MAX_WIDTH);
  GB_REQUIRE(n_jobs >= 0 && n_slots >= 0, GB_E_ARG, "bad n_jobs/n_slots");
  if (n_jobs == 0) return GB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  minmax_init_kernel<float><<<n_jobs, 128, 0, st>>>(jobs, n_out, minmax_ws);
  const int chunks = (max_rows + ROWS_PER_CTA - 1) / ROWS_PER_CTA;
  for (int j0 = 0; chunks > 0 && j0 < n_jobs; j0 += MAX_GRID_Y)
    minmax_reduce_kernel<float><<<dim3(chunks, min(MAX_GRID_Y, n_jobs - j0)), THREADS, 0, st>>>(jobs, j0, y, n_out, minmax_ws);
  minmax_finalize_kernel<<<n_jobs, 128, 0, st>>>(jobs, n_out, minmax_ws, scale, offset);
  GB_CUDA_CHECK(cudaGetLastError());
  return GB_OK;
}

int gb_minmax_f64(const gb_job* jobs, int32_t n_jobs, int32_t max_rows, const double* y, int32_t n_out, double* minmax,
                  int32_t n_slots, void* stream) {
  GB_REQUIRE(jobs && y && minmax, GB_E_ARG, "jobs/y/minmax must be non-NULL");
  GB_REQUIRE(n_out >= 1 && n_out <= GB_MAX_WIDTH, GB_E_SHAPE, "n_out=%d outside [1,%d]", n_out, GB_MAX_WIDTH);
  GB_REQUIRE(n_jobs >= 0 && n_slots >= 0, GB_E_ARG, "bad n_jobs/n_slots");
  if (n_jobs == 0) return GB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  minmax_init_kernel<double><<<n_jobs, 128, 0, st>>>(jobs, n_out, minmax);
  const int chunks = (max_rows + ROWS_PER_CTA - 1) / ROWS_PER_CTA;
  for (int j0 = 0; chunks > 0 && j0 < n_jobs; j0 += MAX_GRID_Y)
    minmax_reduce_kernel<double><<<dim3(chunks, min(MAX_GRID_Y, n_jobs - j0)), THREADS, 0, st>>>(jobs, j0, y, n_out, minmax);
  GB_CUDA_CHECK(cudaGetLastError());
  return GB_OK;
}

int gb_thresholds(const gb_job* jobs, int32_t n_jobs, int32_t max_rows, const float* tag_unscaled,
                  const float* total_scaled, int32_t n_out, int32_t window, float* feat_thr, float* agg_thr,
                  int32_t n_slots, void* stream) {
  return thresholds_launch<float>(jobs, n_jobs, max_rows, tag_unscaled, total_scaled, n_out, window, feat_thr, agg_thr, n_slots, stream);
}

int gb_thresholds_f64(const gb_job* jobs, int32_t n_jobs, int32_t max_rows, const double* tag_unscaled,
                      const double* total_scaled, int32_t n_out, int32_t window, double* feat_thr, double* agg_thr,
                      int32_t n_slots, void* stream) {
  return thresholds_launch<double>(jobs, n_jobs, max_rows, tag_unscaled, total_scaled, n_out, window, feat_thr, agg_thr, n_slots, stream);
}

int gb_cv_moments(const gb_job* jobs, int32_t n_jobs, const float* yhat, const float* y, int32_t n_out, double* out,
                  void* stream) {
  GB_REQUIRE(jobs && yhat && y && out, GB_E_ARG, "jobs/yhat/y/out must be non-NULL");
  GB_REQUIRE(n_out >= 1, GB_E_SHAPE, "n_out=%d must be >= 1", n_out);
  GB_REQUIRE(n_jobs >= 0, GB_E_ARG, "bad n_jobs");
  if (n_jobs == 0) return GB_OK;
  cv_moments_kernel<<<n_jobs, THREADS, 0, (cudaStream_t)stream>>>(jobs, yhat, y, n_out, out);
  GB_CUDA_CHECK(cudaGetLastError());
  return GB_OK;
}

}  // extern "C"
