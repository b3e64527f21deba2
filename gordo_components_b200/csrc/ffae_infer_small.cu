// K1+K4, variant 3: fused Dense-stack forward + anomaly score for NARROW stacks (every width <= 16: the 4- and 8-tag models of
// the reference's own tests and load test, benchmarks/test_ml_server.py:23, tests/conftest.py:80-82).
//
// These nets are a few hundred FLOP per row: the path is purely HBM-bound (6 arrays of 4*T bytes + 3 scalars per row) and the
// 128-row register-tiled kernel of ffae_infer_fma.cu spends its time in barriers with most threads idle.  Here ONE THREAD
// OWNS ONE ROW: the row's activations stay in registers across all layers, the weights are warp-broadcast 128-bit shared-memory
// reads (Keras kernel layout [in][out] is already the broadcast-friendly one), there is no barrier inside the row loop, and
// because a row is 16-64 contiguous bytes, consecutive threads read and write consecutive memory (vector accesses, fully
// coalesced).  Exact fp32 FFMA arithmetic; tanh through ex2.approx/rcp.approx (~2e-7 absolute).
//
// Reference arithmetic replaced: keras Dense act(x @ kernel + bias) under Model.predict (gordo/machine/model/models.py:289-300)
// and DiffBasedAnomalyDetector.anomaly (gordo/machine/model/anomaly/diff.py:350-385, 420-444).
#include "gb_common.cuh"

namespace {

constexpr int THREADS = 256;
constexpr int ROWS_PER_THREAD = 4;
constexpr int CHUNK = THREADS * ROWS_PER_THREAD;

struct SmallArgs {
  gb_ffnet net;
  int n_in, n_out;
  long pstride;
  const float* params;
  const gb_job* jobs;
  const float *x, *y, *scale, *feat_thr, *agg_thr;
  float *o_model, *o_ts, *o_tu, *o_tots, *o_totu, *o_conf, *o_totconf;
  const double *x64, *x_scale, *x_offset;  // float64 x and the slot's input scaler (X64 instantiations; x is then unused)
};

__device__ __forceinline__ float fast_tanh(float z) {
  float e, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(2.8853900817779268f * z));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(e + 1.0f));
  return fmaf(-2.0f, r, 1.0f);
}
__device__ __forceinline__ float act_apply(int act, float z) { return act == GB_ACT_TANH ? fast_tanh(z) : gb::apply_act(act, z); }

// row of T floats <-> registers (zero padded to W); vector path when the row is a whole number of float4
template <int W>
__device__ __forceinline__ void load_row(const float* __restrict__ p, int T, float* v) {
  if ((T & 3) == 0) {
#pragma unroll
    for (int c = 0; c < W / 4; ++c) {
      float4 q = make_float4(0.f, 0.f, 0.f, 0.f);
      if (4 * c < T) q = __ldg(reinterpret_cast<const float4*>(p) + c);
      v[4 * c] = q.x; v[4 * c + 1] = q.y; v[4 * c + 2] = q.z; v[4 * c + 3] = q.w;
    }
  } else {
#pragma unroll
    for (int c = 0; c < W; ++c) v[c] = c < T ? __ldg(p + c) : 0.f;
  }
}
// row of T doubles through the slot's input scaler a, b: (float)(x * a + b), two roundings in double and one to float as
// gb_affine_f64 computes it; zero padded to W
template <int W>
__device__ __forceinline__ void load_row_x64(const double* __restrict__ p, const double* __restrict__ xa, const double* __restrict__ xb, int T,
                                             float* v) {
#pragma unroll
  for (int c = 0; c < W; ++c) v[c] = c < T ? (float)__dadd_rn(__dmul_rn(__ldg(p + c), __ldg(xa + c)), __ldg(xb + c)) : 0.f;
}
template <int W>
__device__ __forceinline__ void store_row(float* __restrict__ p, int T, const float* v) {
  if ((T & 3) == 0) {
#pragma unroll
    for (int c = 0; c < W / 4; ++c)
      if (4 * c < T) __stcs(reinterpret_cast<float4*>(p) + c, make_float4(v[4 * c], v[4 * c + 1], v[4 * c + 2], v[4 * c + 3]));  // streaming: written once
  } else {
#pragma unroll
    for (int c = 0; c < W; ++c)
      if (c < T) p[c] = v[c];
  }
}

template <int W, bool X64>
__global__ void __launch_bounds__(THREADS) ffae_infer_small_kernel(const SmallArgs a) {
  __shared__ __align__(16) float sW[GB_MAX_LAYERS][W][W];  // [layer][k][n], zero padded
  __shared__ __align__(16) float sB[GB_MAX_LAYERS][W];
  __shared__ float sScale[W], sRthr[W];
  const gb_job job = a.jobs[blockIdx.y];
  const int row0 = blockIdx.x * CHUNK;
  if (row0 >= job.n_rows) return;
  const int tid = threadIdx.x, L = a.net.n_layers, T_in = a.n_in, T = a.n_out;
  const float* P = a.params + (long)job.slot * a.pstride;
  {
    int pofs = 0;
    for (int l = 0; l < L; ++l) {
      const int K = a.net.dims[l], N = a.net.dims[l + 1];
      for (int i = tid; i < W * W; i += THREADS) {
        const int k = i / W, n = i - k * W;
        sW[l][k][n] = (k < K && n < N) ? __ldg(P + pofs + k * N + n) : 0.f;
      }
      for (int n = tid; n < W; n += THREADS) sB[l][n] = n < N ? __ldg(P + pofs + K * N + n) : 0.f;
      pofs += K * N + N;
    }
    for (int n = tid; n < W; n += THREADS) {
      sScale[n] = (a.scale && n < T) ? __ldg(a.scale + (long)job.slot * T + n) : 0.f;
      sRthr[n] = (a.feat_thr && n < T) ? 1.0f / __ldg(a.feat_thr + (long)job.slot * T + n) : 0.f;
    }
  }
  __syncthreads();
  const bool has_y = a.y != nullptr;
  const float inv_t = 1.0f / (float)T;
  const float ragg = a.agg_thr ? 1.0f / __ldg(a.agg_thr + job.slot) : 0.f;
  const int row_end = min(job.n_rows, row0 + CHUNK);
  for (int r = row0 + tid; r < row_end; r += THREADS) {
    float act[W];
    if constexpr (X64)
      load_row_x64<W>(a.x64 + (job.x_row + r) * (long)T_in, a.x_scale + (long)job.slot * T_in, a.x_offset + (long)job.slot * T_in, T_in, act);
    else
      load_row<W>(a.x + (job.x_row + r) * (long)T_in, T_in, act);
    for (int l = 0; l < L; ++l) {
      float z[W];
#pragma unroll
      for (int n = 0; n < W; ++n) z[n] = sB[l][n];
#pragma unroll
      for (int k = 0; k < W; ++k) {
        const float ak = act[k];
#pragma unroll
        for (int n4 = 0; n4 < W / 4; ++n4) {
          const float4 w = *reinterpret_cast<const float4*>(&sW[l][k][4 * n4]);  // same address in every lane: one broadcast
          z[4 * n4] = fmaf(ak, w.x, z[4 * n4]);
          z[4 * n4 + 1] = fmaf(ak, w.y, z[4 * n4 + 1]);
          z[4 * n4 + 2] = fmaf(ak, w.z, z[4 * n4 + 2]);
          z[4 * n4 + 3] = fmaf(ak, w.w, z[4 * n4 + 3]);
        }
      }
      const int N = a.net.dims[l + 1], fn = a.net.act[l];
#pragma unroll
      for (int n = 0; n < W; ++n) act[n] = n < N ? act_apply(fn, z[n]) : 0.f;
    }
    const long orow = job.out_row + r;
    store_row<W>(a.o_model + orow * T, T, act);
    if (has_y) {
      float yv[W], d[W], e[W];
      load_row<W>(a.y + (job.x_row + r) * (long)T, T, yv);
      float su = 0.f, ss = 0.f;
#pragma unroll
      for (int n = 0; n < W; ++n) {
        d[n] = n < T ? fabsf(act[n] - yv[n]) : 0.f;
        e[n] = d[n] * sScale[n];
        su = fmaf(d[n], d[n], su);
        ss = fmaf(e[n], e[n], ss);
      }
      if (a.o_tu) store_row<W>(a.o_tu + orow * T, T, d);
      if (a.o_ts) store_row<W>(a.o_ts + orow * T, T, e);
      if (a.o_conf) {
#pragma unroll
        for (int n = 0; n < W; ++n) e[n] = d[n] * sRthr[n];
        store_row<W>(a.o_conf + orow * T, T, e);
      }
      if (a.o_totu) a.o_totu[orow] = su * inv_t;
      if (a.o_tots) a.o_tots[orow] = ss * inv_t;
      if (a.o_totconf) a.o_totconf[orow] = ss * inv_t * ragg;
    }
  }
}

}  // namespace

extern "C" int gb_ffae_small_supported(const gb_ffnet* net) {
  if (gb::validate_ffnet(net) != GB_OK) return GB_E_SHAPE;
  for (int l = 0; l <= net->n_layers; ++l)
    if (net->dims[l] > 16) {
      gb::set_error("the row-per-thread variant covers stacks whose widths are all <= 16");
      return GB_E_SHAPE;
    }
  return GB_OK;
}

// x_scale == NULL: x is float32.  Otherwise x is float64 and x_scale / x_offset [n_slots][n_in] double are the slot's input scaler.
extern "C" int gb_ffae_infer_score_small(const gb_ffnet* net, const float* params, const gb_job* jobs, int32_t n_jobs, int32_t max_rows,
                                         const void* x, const double* x_scale, const double* x_offset, const float* y, const float* scale, const float* feat_thr, const float* agg_thr,
                                         float* out_model, float* out_tag_scaled, float* out_tag_unscaled, float* out_total_scaled,
                                         float* out_total_unscaled, float* out_conf, float* out_total_conf, void* stream) {
  int rc = gb_ffae_small_supported(net);
  if (rc != GB_OK) return rc;
  SmallArgs a{};
  a.net = *net;
  a.n_in = net->dims[0];
  a.n_out = net->dims[net->n_layers];
  a.pstride = (long)gb_ffnet_param_stride(net);
  const bool x64 = x_scale != nullptr;
  if (x64) {
    a.x64 = static_cast<const double*>(x); a.x_scale = x_scale; a.x_offset = x_offset;
  } else {
    a.x = static_cast<const float*>(x);
  }
  a.params = params; a.jobs = jobs; a.y = y; a.scale = scale; a.feat_thr = feat_thr; a.agg_thr = agg_thr;
  a.o_model = out_model; a.o_ts = out_tag_scaled; a.o_tu = out_tag_unscaled; a.o_tots = out_total_scaled;
  a.o_totu = out_total_unscaled; a.o_conf = out_conf; a.o_totconf = out_total_conf;
  int wmax = 0;
  for (int l = 0; l <= net->n_layers; ++l) wmax = net->dims[l] > wmax ? net->dims[l] : wmax;
  for (int j0 = 0; j0 < n_jobs; j0 += 65535) {  // gridDim.y carries the job index: larger fleets go out as several launches
    a.jobs = jobs + j0;
    const dim3 grid((max_rows + CHUNK - 1) / CHUNK, n_jobs - j0 < 65535 ? n_jobs - j0 : 65535);
    const auto kern = wmax <= 4 ? (x64 ? ffae_infer_small_kernel<4, true> : ffae_infer_small_kernel<4, false>)
                      : wmax <= 8 ? (x64 ? ffae_infer_small_kernel<8, true> : ffae_infer_small_kernel<8, false>)
                                  : (x64 ? ffae_infer_small_kernel<16, true> : ffae_infer_small_kernel<16, false>);
    kern<<<grid, THREADS, 0, (cudaStream_t)stream>>>(a);
  }
  GB_CUDA_CHECK(cudaGetLastError());
  return GB_OK;
}
