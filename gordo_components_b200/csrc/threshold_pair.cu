// gb_thresholds_pair[_f64]: the 6-row and the smoothing-window fold thresholds of a DiffBasedAnomalyDetector in one pass
// (reference diff.py:222-233 and 242-258): rolling(w).min().max() of every tag column and of the aggregate series, for two
// windows w0 and w1, reading each score element once.
//
// The rolling minimum is van Herk / Gil-Werman: with the rows cut into blocks of w (from some origin a),
//   min(x[t-w+1 .. t]) = min(S[t-w+1], P[t])
// where P is the prefix minimum of t's block and S the suffix minimum of the block before it.  One thread walks one column of
// one run of rows in order, keeping P in a register and, per window, a private buffer of w values: at block position r it
// reads S_prev[r+1] (the suffix of the previous block from r+1 on), then stores x in slot r (slot r of S_prev is no longer
// needed), and at the end of a block turns the buffer into that block's suffix minima in place.  Per row and window: one
// buffer read, one write and, amortised, one read-modify-write of the suffix pass, whatever the window.
//
// The buffers live in shared memory when a warp's fit there, and otherwise in a global scratch area the launch allocates on the
// stream.  A run of rows starts wmax rows early (its warm-up) so that its first window is complete.
//
// NaN is carried as -inf: a window holding one has a minimum below the "no window yet" marker -1, so max() skips it as pandas'
// does; every other value is compared exactly as rollmin_max_kernel compares it, so the thresholds are bit for bit
// gb_thresholds' at each window.
#include <math_constants.h>
#include "gb_common.cuh"

namespace {

template <typename T> struct PairBits;
template <> struct PairBits<float> {
  using I = int;
  static __device__ __forceinline__ I bits(float v) { return __float_as_int(v); }
  static __device__ __forceinline__ float nan() { return CUDART_NAN_F; }
  static __device__ __forceinline__ float inf() { return CUDART_INF_F; }
};
template <> struct PairBits<double> {
  using I = long long;
  static __device__ __forceinline__ I bits(double v) { return __double_as_longlong(v); }
  static __device__ __forceinline__ double nan() { return CUDART_NAN; }
  static __device__ __forceinline__ double inf() { return CUDART_INF; }
};

constexpr int MIN_RUN = 1024;         // rows a thread owns (at least 4 * wmax, so the warm-up costs at most a quarter more)
constexpr long SCRATCH_BYTES = 64l << 20;  // global buffers, when a warp's do not fit in shared memory

// slot-wise outputs: -1 marks "no complete window yet"
template <typename T>
__global__ void pair_init_kernel(const gb_job* jobs, int n_jobs, int n_out, T* f0, T* a0, T* f1, T* a1) {
  const int i = blockIdx.x * blockDim.y + threadIdx.y;
  if (i >= n_jobs) return;
  const long s = jobs[i].slot;
  for (int j = threadIdx.x; j < n_out; j += blockDim.x) {
    if (f0) { f0[s * n_out + j] = (T)-1; f1[s * n_out + j] = (T)-1; }
  }
  if (threadIdx.x == 0 && a0) { a0[s] = (T)-1; a1[s] = (T)-1; }
}

template <typename T>
__global__ void pair_finalize_kernel(const gb_job* jobs, int n_jobs, int n_out, T* f0, T* a0, T* f1, T* a1) {
  const int i = blockIdx.x * blockDim.y + threadIdx.y;
  if (i >= n_jobs) return;
  const long s = jobs[i].slot;
  const auto fix = [](T* p) { if (*p < (T)0) *p = PairBits<T>::nan(); };  // fewer rows than the window: pandas gives NaN
  for (int j = threadIdx.x; j < n_out; j += blockDim.x) {
    if (f0) { fix(&f0[s * n_out + j]); fix(&f1[s * n_out + j]); }
  }
  if (threadIdx.x == 0 && a0) { fix(&a0[s]); fix(&a1[s]); }
}

// The state of one window's rolling minimum along one column.
template <typename T>
struct Roll {
  T* buf;         // w slots, `stride` elements apart
  long stride;
  int w, r;       // window, position in the current block
  long emit;      // first row whose window is complete and inside this thread's run
  T p, best;

  __device__ __forceinline__ void push(long t, T x) {
    p = r == 0 ? x : (x < p ? x : p);
    if (t >= emit) {
      const T s = r + 1 < w ? buf[(r + 1) * stride] : PairBits<T>::inf();
      const T m = s < p ? s : p;
      best = m > best ? m : best;
    }
    buf[r * stride] = x;
    if (++r == w) {  // block complete: its suffix minima, in place
      T c = x;
#pragma unroll 4
      for (int q = w - 2; q >= 0; --q) {
        const T v = buf[q * stride];
        c = v < c ? v : c;
        buf[q * stride] = c;
      }
      r = 0;
    }
  }

  __device__ __forceinline__ void publish(T* out) const {
    const T b = best + (T)0;  // -0.0 -> +0.0: as an integer -0.0 would never beat the -1 marker
    if (b >= (T)0) atomicMax(reinterpret_cast<typename PairBits<T>::I*>(out), PairBits<T>::bits(b));
  }
};

template <typename T>
constexpr int unroll() { return sizeof(T) == 4 ? 8 : 4; }  // loads in flight per thread (without spilling for double)

// Item i (grid-stride) = (job, run, column) with the column fastest, so a warp reads neighbouring columns of one row.  Columns
// [0, n_out) are the tags, column n_out the aggregate series; [c_lo, c_hi) are those requested.  Windows of 0 are skipped.
template <typename T>
__global__ void __launch_bounds__(256) pair_kernel(const gb_job* jobs, long n_items, int runs, int run_rows, int c_lo, int n_c,
                                                   const T* __restrict__ tag, const T* __restrict__ total, int n_out, int w0, int w1,
                                                   T* f0, T* a0, T* f1, T* a1, T* scratch) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const long n_threads = (long)gridDim.x * blockDim.x;
  const long tid = (long)blockIdx.x * blockDim.x + threadIdx.x;
  T* base;
  long stride;
  if (scratch) { base = scratch + tid; stride = n_threads; }
  else { base = reinterpret_cast<T*>(smem_raw) + threadIdx.x; stride = blockDim.x; }
  const int wmax = w0 > w1 ? w0 : w1;
  for (long item = tid; item < n_items; item += n_threads) {
    const int c = c_lo + (int)(item % n_c);
    const long jr = item / n_c;
    const gb_job job = jobs[jr / runs];
    const long t0 = (jr % runs) * (long)run_rows;
    if (t0 >= job.n_rows) continue;
    const long t1 = t0 + run_rows < job.n_rows ? t0 + run_rows : job.n_rows;
    const long a = t0 - wmax > 0 ? t0 - wmax : 0;  // the warm-up: every window ending in [t0, t1) is read whole
    const bool agg = c == n_out;
    const T* src = agg ? total + job.out_row : tag + job.out_row * (long)n_out + c;
    const long ld = agg ? 1 : n_out;
    Roll<T> r0{base, stride, w0, 0, t0 > a + w0 - 1 ? t0 : a + w0 - 1, (T)0, (T)-1};
    Roll<T> r1{base + (long)w0 * stride, stride, w1, 0, t0 > a + w1 - 1 ? t0 : a + w1 - 1, (T)0, (T)-1};
    for (long t = a; t < t1; t += unroll<T>()) {
      constexpr int UNROLL = unroll<T>();
      T v[UNROLL];
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) v[u] = t + u < t1 ? __ldg(src + (t + u) * ld) : (T)0;
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        if (t + u < t1) {
          const T x = v[u] == v[u] ? v[u] : -PairBits<T>::inf();  // NaN sorts below every score
          if (w0) r0.push(t + u, x);
          if (w1) r1.push(t + u, x);
        }
      }
    }
    const long s = job.slot;
    if (w0) r0.publish(agg ? a0 + s : f0 + s * n_out + c);
    if (w1) r1.publish(agg ? a1 + s : f1 + s * n_out + c);
  }
}

// The launch shape of the buffers: threads per CTA and dynamic shared memory, or 0 threads when a warp's buffers exceed the
// shared memory one CTA may have (the global scratch path).
struct PairPlan {
  int threads;
  size_t smem;
};

PairPlan pair_plan(size_t bytes_per_thread) {
  int dev = 0, sm_smem = 0, optin = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sm_smem, cudaDevAttrMaxSharedMemoryPerMultiprocessor, dev);
  cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  PairPlan best{0, 0};
  long best_resident = 0;
  for (int warps = 1; warps <= 8; warps *= 2) {  // the CTA size that keeps the most threads resident per SM
    const size_t bytes = (size_t)warps * 32 * bytes_per_thread;
    if (bytes > (size_t)optin) break;
    long ctas = (long)sm_smem / (long)(bytes + 1024);
    ctas = ctas < 32 ? ctas : 32;
    ctas = ctas < 64 / warps ? ctas : 64 / warps;
    if (ctas * warps * 32 >= best_resident) { best_resident = ctas * warps * 32; best = {warps * 32, bytes}; }
  }
  return best;
}

template <typename T>
int thresholds_pair_launch(const gb_job* jobs, int32_t n_jobs, int32_t max_rows, const T* tag_unscaled, const T* total_scaled,
                           int32_t n_out, int32_t w0, int32_t w1, T* feat_thr0, T* agg_thr0, T* feat_thr1, T* agg_thr1,
                           int32_t n_slots, void* stream) {
  GB_REQUIRE(jobs, GB_E_ARG, "jobs must be non-NULL");
  GB_REQUIRE((tag_unscaled != nullptr) == (feat_thr0 != nullptr) && (feat_thr0 != nullptr) == (feat_thr1 != nullptr), GB_E_ARG,
             "tag_unscaled, feat_thr0 and feat_thr1 go together");
  GB_REQUIRE((total_scaled != nullptr) == (agg_thr0 != nullptr) && (agg_thr0 != nullptr) == (agg_thr1 != nullptr), GB_E_ARG,
             "total_scaled, agg_thr0 and agg_thr1 go together");
  GB_REQUIRE(n_out >= 1 && n_out <= GB_MAX_WIDTH, GB_E_SHAPE, "n_out=%d outside [1,%d]", n_out, GB_MAX_WIDTH);
  GB_REQUIRE(w0 >= 1, GB_E_ARG, "w0=%d must be >= 1", w0);
  GB_REQUIRE(w1 >= 1, GB_E_ARG, "w1=%d must be >= 1", w1);
  GB_REQUIRE(max_rows >= 0, GB_E_ARG, "max_rows=%d must be >= 0", max_rows);
  GB_REQUIRE(n_jobs >= 0, GB_E_ARG, "n_jobs=%d must be >= 0", n_jobs);
  GB_REQUIRE(n_slots >= 0, GB_E_ARG, "n_slots=%d must be >= 0", n_slots);
  if (n_jobs == 0) return GB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const dim3 small(32, 8);
  const int small_grid = (n_jobs + 7) / 8;
  pair_init_kernel<T><<<small_grid, small, 0, st>>>(jobs, n_jobs, n_out, feat_thr0, agg_thr0, feat_thr1, agg_thr1);
  // a window longer than every job has no complete window anywhere: its thresholds stay NaN and it needs no buffer
  const int k0 = w0 <= max_rows ? w0 : 0, k1 = w1 <= max_rows ? w1 : 0;
  const int c_lo = tag_unscaled ? 0 : n_out, c_hi = total_scaled ? n_out + 1 : n_out;
  if ((k0 || k1) && c_hi > c_lo) {
    const int wmax = k0 > k1 ? k0 : k1;
    const int run_rows = 4 * wmax > MIN_RUN ? 4 * wmax : MIN_RUN;
    const int runs = (max_rows + run_rows - 1) / run_rows;
    const long n_items = (long)n_jobs * runs * (c_hi - c_lo);
    const size_t per_thread = (size_t)(k0 + k1) * sizeof(T);
    const PairPlan plan = pair_plan(per_thread);
    if (plan.threads) {
      GB_CUDA_CHECK(cudaFuncSetAttribute(pair_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)plan.smem));
      const long blocks = (n_items + plan.threads - 1) / plan.threads;
      pair_kernel<T><<<(unsigned)blocks, plan.threads, plan.smem, st>>>(jobs, n_items, runs, run_rows, c_lo, c_hi - c_lo, tag_unscaled,
                                                                       total_scaled, n_out, k0, k1, feat_thr0, agg_thr0, feat_thr1,
                                                                       agg_thr1, nullptr);
    } else {
      long threads = SCRATCH_BYTES / (long)per_thread;
      threads = threads > 32 ? threads : 32;
      threads = threads < n_items ? threads : n_items;
      const long blocks = (threads + 127) / 128;
      T* scratch = nullptr;
      GB_CUDA_CHECK(cudaMallocAsync(reinterpret_cast<void**>(&scratch), (size_t)blocks * 128 * per_thread, st));
      pair_kernel<T><<<(unsigned)blocks, 128, 0, st>>>(jobs, n_items, runs, run_rows, c_lo, c_hi - c_lo, tag_unscaled, total_scaled, n_out,
                                                      k0, k1, feat_thr0, agg_thr0, feat_thr1, agg_thr1, scratch);
      GB_CUDA_CHECK(cudaFreeAsync(scratch, st));
    }
  }
  pair_finalize_kernel<T><<<small_grid, small, 0, st>>>(jobs, n_jobs, n_out, feat_thr0, agg_thr0, feat_thr1, agg_thr1);
  GB_CUDA_CHECK(cudaGetLastError());
  return GB_OK;
}

}  // namespace

extern "C" {

int gb_thresholds_pair(const gb_job* jobs, int32_t n_jobs, int32_t max_rows, const float* tag_unscaled, const float* total_scaled,
                       int32_t n_out, int32_t w0, int32_t w1, float* feat_thr0, float* agg_thr0, float* feat_thr1, float* agg_thr1,
                       int32_t n_slots, void* stream) {
  return thresholds_pair_launch<float>(jobs, n_jobs, max_rows, tag_unscaled, total_scaled, n_out, w0, w1, feat_thr0, agg_thr0, feat_thr1,
                                       agg_thr1, n_slots, stream);
}

int gb_thresholds_pair_f64(const gb_job* jobs, int32_t n_jobs, int32_t max_rows, const double* tag_unscaled, const double* total_scaled,
                           int32_t n_out, int32_t w0, int32_t w1, double* feat_thr0, double* agg_thr0, double* feat_thr1,
                           double* agg_thr1, int32_t n_slots, void* stream) {
  return thresholds_pair_launch<double>(jobs, n_jobs, max_rows, tag_unscaled, total_scaled, n_out, w0, w1, feat_thr0, agg_thr0, feat_thr1,
                                        agg_thr1, n_slots, stream);
}

}  // extern "C"
