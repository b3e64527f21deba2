// Row permutations and the float32 MinMax inverse of the batched K-fold build.
//   gb_gather_rows         : dst[out_row + p] = src[x_row + row_map[p]] for every job (one map shared by all jobs), 4- or
//                            8-byte elements, optionally narrowing float64 -> float32 on the way
//   gb_gather_rows_ragged  : the same with a map per job, row_map[map_ofs[job] + p] (machines of different lengths in one bucket)
//   gb_minmax_inverse_f32  : sklearn's MinMaxScaler.inverse_transform of a float32 prediction (TransformedTargetRegressor.predict)
// Both are HBM-bound single passes: a grid-stride loop over the job's (row, unit) pairs, the job index on gridDim.y.
#include "gb_common.cuh"
#include "postprocess.cuh"

namespace {

constexpr int THREADS = 256;
constexpr int MAX_GRID_Y = 65535;  // gridDim.y carries the job index: larger fleets go out as several launches (job0 = first job)

// Same-size copy of rows of `units` elements of U (uint4 when a row is a whole number of 16-byte units and both arrays are aligned).
// PER_JOB: job i reads its own map at map + map_ofs[i]; map_ofs comes last so the shared-map kernels keep their parameter offsets.
template <typename U, bool PER_JOB>
__global__ void __launch_bounds__(THREADS) gather_copy_kernel(const gb_job* __restrict__ jobs, int job0, const int32_t* __restrict__ map,
                                                              const U* __restrict__ src, U* __restrict__ dst, int units,
                                                              const int64_t* __restrict__ map_ofs) {
  const gb_job job = jobs[job0 + blockIdx.y];
  if (PER_JOB) map += map_ofs[job0 + blockIdx.y];
  const long total = (long)job.n_rows * units;
  const U* s = src + job.x_row * units;
  U* d = dst + job.out_row * units;
  for (long i = (long)blockIdx.x * THREADS + threadIdx.x; i < total; i += (long)gridDim.x * THREADS) {
    const int p = (int)(i / units);
    const int c = (int)(i - (long)p * units);
    d[i] = __ldg(s + (long)__ldg(map + p) * units + c);
  }
}

// float64 -> float32 (round to nearest), two elements per step when rows hold an even number of them.  PER_JOB as gather_copy_kernel.
template <int V, bool PER_JOB>
__global__ void __launch_bounds__(THREADS) gather_narrow_kernel(const gb_job* __restrict__ jobs, int job0, const int32_t* __restrict__ map,
                                                                const double* __restrict__ src, float* __restrict__ dst, int n_cols,
                                                                const int64_t* __restrict__ map_ofs) {
  const gb_job job = jobs[job0 + blockIdx.y];
  if (PER_JOB) map += map_ofs[job0 + blockIdx.y];
  const int units = n_cols / V;
  const long total = (long)job.n_rows * units;
  const double* s = src + job.x_row * n_cols;
  float* d = dst + job.out_row * n_cols;
  for (long i = (long)blockIdx.x * THREADS + threadIdx.x; i < total; i += (long)gridDim.x * THREADS) {
    const int p = (int)(i / units);
    const int c = (int)(i - (long)p * units);
    const double* from = s + (long)__ldg(map + p) * n_cols + c * V;
    if (V == 2) {
      const double2 v = __ldg(reinterpret_cast<const double2*>(from));
      reinterpret_cast<float2*>(d)[i] = make_float2(__double2float_rn(v.x), __double2float_rn(v.y));
    } else {
      d[i] = __double2float_rn(__ldg(from));
    }
  }
}

// X -= min_; X /= scale_ on a float32 array with float64 attributes (gb_post::minmax_inverse).
__global__ void __launch_bounds__(THREADS) minmax_inverse_kernel(const gb_job* __restrict__ jobs, int job0, const float* __restrict__ p, int n_cols,
                                                                 const double* __restrict__ scale, const double* __restrict__ mn,
                                                                 float* __restrict__ out32, double* __restrict__ out64) {
  const gb_job job = jobs[job0 + blockIdx.y];
  const long total = (long)job.n_rows * n_cols;
  const float* src = p + job.x_row * n_cols;
  const long o = job.out_row * n_cols;
  const double* js = scale + (long)job.slot * n_cols;
  const double* jm = mn + (long)job.slot * n_cols;
  for (long i = (long)blockIdx.x * THREADS + threadIdx.x; i < total; i += (long)gridDim.x * THREADS) {
    const int c = (int)(i % n_cols);
    const float v = gb_post::minmax_inverse(__ldg(src + i), jm + c, js + c);
    if (out32) out32[o + i] = v;
    if (out64) out64[o + i] = (double)v;
  }
}

inline dim3 grid_for(long per_job, int n_jobs_left) {
  long bx = (per_job + THREADS * 4L - 1) / (THREADS * 4L);
  bx = bx < 1 ? 1 : (bx > 1184 ? 1184 : bx);
  return dim3((unsigned)bx, n_jobs_left < MAX_GRID_Y ? n_jobs_left : MAX_GRID_Y);
}

// Both gather entry points: every argument check, then the launches (PER_JOB: a map per job, at row_map + map_ofs[job]).
template <bool PER_JOB>
int gather_launch(const gb_job* jobs, int32_t n_jobs, int32_t max_rows, const int32_t* row_map, const int64_t* map_ofs, const void* src,
                  int32_t n_cols, int32_t elem_bytes, int32_t to_f32, void* dst, void* stream) {
  GB_REQUIRE(jobs && row_map && src && dst, GB_E_ARG, "jobs/row_map/src/dst must be non-NULL");
  GB_REQUIRE(elem_bytes == 4 || elem_bytes == 8, GB_E_ARG, "elem_bytes=%d must be 4 or 8", elem_bytes);
  GB_REQUIRE(!to_f32 || elem_bytes == 8, GB_E_ARG, "to_f32 narrows 8-byte (float64) elements");
  GB_REQUIRE(n_cols >= 1 && max_rows >= 0 && n_jobs >= 0, GB_E_ARG, "n_cols=%d max_rows=%d n_jobs=%d", n_cols, max_rows, n_jobs);
  GB_REQUIRE(!PER_JOB || map_ofs, GB_E_ARG, "map_ofs must be non-NULL");
  if (n_jobs == 0 || max_rows == 0) return GB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const uintptr_t both = (uintptr_t)src | (uintptr_t)dst;
  for (int j0 = 0; j0 < n_jobs; j0 += MAX_GRID_Y) {
    if (to_f32) {
      const bool pair = n_cols % 2 == 0 && (uintptr_t)src % 16 == 0 && (uintptr_t)dst % 8 == 0;
      const dim3 grid = grid_for((long)max_rows * (pair ? n_cols / 2 : n_cols), n_jobs - j0);
      if (pair) gather_narrow_kernel<2, PER_JOB><<<grid, THREADS, 0, st>>>(jobs, j0, row_map, (const double*)src, (float*)dst, n_cols, map_ofs);
      else gather_narrow_kernel<1, PER_JOB><<<grid, THREADS, 0, st>>>(jobs, j0, row_map, (const double*)src, (float*)dst, n_cols, map_ofs);
      continue;
    }
    const long row_bytes = (long)n_cols * elem_bytes;
    if (row_bytes % 16 == 0 && both % 16 == 0) {
      const int units = (int)(row_bytes / 16);
      gather_copy_kernel<uint4, PER_JOB><<<grid_for((long)max_rows * units, n_jobs - j0), THREADS, 0, st>>>(jobs, j0, row_map, (const uint4*)src,
                                                                                                            (uint4*)dst, units, map_ofs);
    } else if (elem_bytes == 8) {
      gather_copy_kernel<unsigned long long, PER_JOB><<<grid_for((long)max_rows * n_cols, n_jobs - j0), THREADS, 0, st>>>(
          jobs, j0, row_map, (const unsigned long long*)src, (unsigned long long*)dst, n_cols, map_ofs);
    } else {
      gather_copy_kernel<unsigned int, PER_JOB><<<grid_for((long)max_rows * n_cols, n_jobs - j0), THREADS, 0, st>>>(
          jobs, j0, row_map, (const unsigned int*)src, (unsigned int*)dst, n_cols, map_ofs);
    }
  }
  GB_CUDA_CHECK(cudaGetLastError());
  return GB_OK;
}

}  // namespace

extern "C" int gb_gather_rows(const gb_job* jobs, int32_t n_jobs, int32_t max_rows, const int32_t* row_map, const void* src, int32_t n_cols,
                              int32_t elem_bytes, int32_t to_f32, void* dst, void* stream) {
  return gather_launch<false>(jobs, n_jobs, max_rows, row_map, nullptr, src, n_cols, elem_bytes, to_f32, dst, stream);
}

extern "C" int gb_gather_rows_ragged(const gb_job* jobs, int32_t n_jobs, int32_t max_rows, const int32_t* row_map, const int64_t* map_ofs,
                                     const void* src, int32_t n_cols, int32_t elem_bytes, int32_t to_f32, void* dst, void* stream) {
  return gather_launch<true>(jobs, n_jobs, max_rows, row_map, map_ofs, src, n_cols, elem_bytes, to_f32, dst, stream);
}

extern "C" int gb_minmax_inverse_f32(const gb_job* jobs, int32_t n_jobs, int32_t max_rows, const float* p, int32_t n_cols, const double* scale,
                                     const double* min_, float* out_f32, double* out_f64, void* stream) {
  GB_REQUIRE(jobs && p && scale && min_, GB_E_ARG, "jobs/p/scale/min_ must be non-NULL");
  GB_REQUIRE(out_f32 || out_f64, GB_E_ARG, "no output requested");
  GB_REQUIRE(n_cols >= 1 && max_rows >= 0 && n_jobs >= 0, GB_E_ARG, "n_cols=%d max_rows=%d n_jobs=%d", n_cols, max_rows, n_jobs);
  if (n_jobs == 0 || max_rows == 0) return GB_OK;
  for (int j0 = 0; j0 < n_jobs; j0 += MAX_GRID_Y)
    minmax_inverse_kernel<<<grid_for((long)max_rows * n_cols, n_jobs - j0), THREADS, 0, (cudaStream_t)stream>>>(jobs, j0, p, n_cols, scale, min_,
                                                                                                             out_f32, out_f64);
  GB_CUDA_CHECK(cudaGetLastError());
  return GB_OK;
}
