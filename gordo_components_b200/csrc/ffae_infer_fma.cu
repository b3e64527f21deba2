// K1+K4, variant 1: fused Dense-stack forward + anomaly score on the fp32 CUDA cores.
//
// Generic in the architecture (any widths <= GB_MAX_WIDTH, any supported activation); this is the
// path for the architectures the tensor-core kernel (ffae_infer_tc.cu) does not cover, and the exact-fp32
// cross-check for it.  One CTA owns one job chunk: the slot's weights are copied once into a padded
// shared-memory image, then 128-row tiles stream through: X tile -> smem, every layer is a register-tiled
// [128 x K] x [K x N] product out of shared memory (4 rows x 4 cols per thread, rows interleaved by 32 so
// activation reads are conflict-free LDS.128 and weight reads are warp broadcasts), activations ping-pong
// between two smem buffers, and the epilogue forms all score outputs from the last buffer with coalesced,
// 128-bit global accesses.
//
// Reference arithmetic replaced: keras Dense act(x @ kernel + bias) under Model.predict
// (gordo/machine/model/models.py:289-300) and DiffBasedAnomalyDetector.anomaly
// (gordo/machine/model/anomaly/diff.py:350-385, 420-444).
#include "gb_common.cuh"

namespace {

constexpr int THREADS = 256;
constexpr int NWARPS = THREADS / 32;

struct Args {
  gb_ffnet net;
  gb::FFImage im;
  int pitch;        // floats between consecutive rows of an activation buffer (pitch/4 odd)
  int wfloats;      // floats reserved for weights in smem
  int resident;     // all layers resident (1) or staged layer by layer (0)
  int col_block;    // staged: output columns of a layer staged at a time (>= every padded width unless a layer is too large)
  int n_in, n_out;
  int rows_per_chunk;
  long pstride;
  const float* params;
  const gb_job* jobs;
  const float *x, *y, *scale, *feat_thr, *agg_thr;
  float *o_model, *o_ts, *o_tu, *o_tots, *o_totu, *o_conf, *o_totconf;
  const double *x64, *x_scale, *x_offset;  // float64 x and the slot's input scaler (X64 instantiations; x is then unused)
};

// output columns [c0, c0 + nb) of layer l as a padded [Kp][nb] image followed by their nb biases
__device__ __forceinline__ void stage_layer(float* dst, const float* P, const Args& a, int l, int c0, int nb, int tid) {
  const int K = a.net.dims[l], N = a.net.dims[l + 1], Kp = a.im.kp[l];
  const float* Wg = P + a.im.pofs[l];
  const float* bg = Wg + K * N;
  for (int idx = tid; idx < Kp * nb; idx += THREADS) {
    const int k = idx / nb, n = c0 + idx - k * nb;
    dst[idx] = (k < K && n < N) ? __ldg(Wg + k * N + n) : 0.f;
  }
  for (int n = tid; n < nb; n += THREADS) dst[Kp * nb + n] = c0 + n < N ? __ldg(bg + c0 + n) : 0.f;
}

// RT row groups of 32 per thread: tiles of 128 rows (RT = 4) for the usual stacks, 64 / 32 rows when wide layers (up to 256: the
// defaults of feedforward_model / feedforward_symmetric) leave less shared memory for the activation buffers.  BLOCKED: staged
// layers go in blocks of a.col_block output columns (only with 32-row tiles, for layers too large to stage whole); a separate
// instantiation so that every other plan runs the single-block code.  X64: x is float64 and the slot's input scaler is applied as
// it is read, x' = (float)(x * x_scale + x_offset) with two roundings in double and one to float, as gb_affine_f64 computes it.
template <int RT, bool BLOCKED, bool X64>
__global__ void __launch_bounds__(THREADS) ffae_infer_fma_kernel(const Args a) {
  constexpr int ROWS = 32 * RT;
  extern __shared__ __align__(16) float smem[];
  float* sW = smem;
  float* buf0 = sW + a.wfloats;
  float* buf1 = buf0 + ROWS * a.pitch;
  float* rowsum = buf1 + ROWS * a.pitch;  // [2][ROWS]

  const gb_job job = a.jobs[blockIdx.y];
  const int row_begin = blockIdx.x * a.rows_per_chunk;
  if (row_begin >= job.n_rows) return;
  const int row_end = min(job.n_rows, row_begin + a.rows_per_chunk);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* P = a.params + (long)job.slot * a.pstride;
  const int pitch = a.pitch, n_in = a.n_in, n_out = a.n_out, L = a.net.n_layers;

  if (a.resident) {
    for (int l = 0; l < L; ++l) stage_layer(sW + a.im.wofs[l], P, a, l, 0, a.im.np[l], tid);
  }
  __syncthreads();

  for (int tile = row_begin; tile < row_end; tile += ROWS) {
    const int nrows = min(ROWS, row_end - tile);
    // ---- X tile -> buf0[r][k], zero padded -------------------------------------------------
    if constexpr (X64) {
      const double* xg = a.x64 + (job.x_row + tile) * (long)n_in;
      const double* xa = a.x_scale + (long)job.slot * n_in;
      const double* xb = a.x_offset + (long)job.slot * n_in;
      const int Tp = a.im.kp[0];
      for (int idx = tid; idx < ROWS * Tp; idx += THREADS) {
        const int r = idx / Tp, k = idx - r * Tp;
        buf0[r * pitch + k] = (r < nrows && k < n_in) ? (float)__dadd_rn(__dmul_rn(__ldg(xg + (long)r * n_in + k), __ldg(xa + k)), __ldg(xb + k)) : 0.f;
      }
    } else {
      const float* xg = a.x + (job.x_row + tile) * (long)n_in;
      const int Tp = a.im.kp[0];
      if ((n_in & 3) == 0) {
        const int T4 = n_in >> 2;
        for (int idx = tid; idx < ROWS * T4; idx += THREADS) {
          const int r = idx / T4, k4 = idx - r * T4;
          float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
          if (r < nrows) v = __ldg(reinterpret_cast<const float4*>(xg + (long)r * n_in) + k4);
          *reinterpret_cast<float4*>(buf0 + r * pitch + 4 * k4) = v;
        }
      } else {
        for (int idx = tid; idx < ROWS * Tp; idx += THREADS) {
          const int r = idx / Tp, k = idx - r * Tp;
          buf0[r * pitch + k] = (r < nrows && k < n_in) ? __ldg(xg + (long)r * n_in + k) : 0.f;
        }
      }
    }
    __syncthreads();

    // ---- Dense layers ------------------------------------------------------------------------
    float* in = buf0;
    float* out = buf1;
    for (int l = 0; l < L; ++l) {
      const int Kp = a.im.kp[l], Np = a.im.np[l], act = a.net.act[l];
      const int cb = BLOCKED ? min(Np, a.col_block) : Np;
      int c0 = 0;
      do {
        const int nb = BLOCKED ? min(cb, Np - c0) : Np;
        const float* Wl;
        if (a.resident) {
          Wl = sW + a.im.wofs[l];
        } else {
          if (BLOCKED && c0 > 0) __syncthreads();  // every warp is done with the previous column block
          stage_layer(sW, P, a, l, c0, nb, tid);
          __syncthreads();
          Wl = sW;
        }
        const float* bl = Wl + Kp * nb;
        for (int task = warp; task < (nb >> 2); task += NWARPS) {
          const int n0 = task << 2;
          const float4 b4 = *reinterpret_cast<const float4*>(bl + n0);
          float4 acc[RT];
#pragma unroll
          for (int i = 0; i < RT; ++i) acc[i] = b4;
          const float* arow = in + lane * pitch;
          const float* wcol = Wl + n0;
          for (int k = 0; k < Kp; k += 4) {
            float4 av[RT];
#pragma unroll
            for (int i = 0; i < RT; ++i) av[i] = *reinterpret_cast<const float4*>(arow + i * 32 * pitch + k);
            const float4 w0 = *reinterpret_cast<const float4*>(wcol + (k + 0) * nb);
            const float4 w1 = *reinterpret_cast<const float4*>(wcol + (k + 1) * nb);
            const float4 w2 = *reinterpret_cast<const float4*>(wcol + (k + 2) * nb);
            const float4 w3 = *reinterpret_cast<const float4*>(wcol + (k + 3) * nb);
#pragma unroll
            for (int i = 0; i < RT; ++i) {
              acc[i].x = fmaf(av[i].x, w0.x, acc[i].x); acc[i].y = fmaf(av[i].x, w0.y, acc[i].y);
              acc[i].z = fmaf(av[i].x, w0.z, acc[i].z); acc[i].w = fmaf(av[i].x, w0.w, acc[i].w);
              acc[i].x = fmaf(av[i].y, w1.x, acc[i].x); acc[i].y = fmaf(av[i].y, w1.y, acc[i].y);
              acc[i].z = fmaf(av[i].y, w1.z, acc[i].z); acc[i].w = fmaf(av[i].y, w1.w, acc[i].w);
              acc[i].x = fmaf(av[i].z, w2.x, acc[i].x); acc[i].y = fmaf(av[i].z, w2.y, acc[i].y);
              acc[i].z = fmaf(av[i].z, w2.z, acc[i].z); acc[i].w = fmaf(av[i].z, w2.w, acc[i].w);
              acc[i].x = fmaf(av[i].w, w3.x, acc[i].x); acc[i].y = fmaf(av[i].w, w3.y, acc[i].y);
              acc[i].z = fmaf(av[i].w, w3.z, acc[i].z); acc[i].w = fmaf(av[i].w, w3.w, acc[i].w);
            }
          }
          // columns past the layer's width stay 0, as in the row-per-thread kernel: their zero weights times an infinite input are
          // NaN, which the next layer would spread over the whole row
          const int n_live = a.net.dims[l + 1] - (c0 + n0);
#pragma unroll
          for (int i = 0; i < RT; ++i) {
            float4 o;
            o.x = gb::apply_act(act, acc[i].x);
            o.y = n_live > 1 ? gb::apply_act(act, acc[i].y) : 0.f;
            o.z = n_live > 2 ? gb::apply_act(act, acc[i].z) : 0.f;
            o.w = n_live > 3 ? gb::apply_act(act, acc[i].w) : 0.f;
            *reinterpret_cast<float4*>(out + (lane + 32 * i) * pitch + c0 + n0) = o;
          }
        }
        c0 += cb;
      } while (BLOCKED && c0 < Np);
      __syncthreads();
      float* t = in; in = out; out = t;
    }

    // ---- epilogue: model output + anomaly scores (in = yhat[r][j]) -----------------------------
    const long orow = job.out_row + tile;
    const bool score = a.y != nullptr;
    const float* yg = score ? a.y + (job.x_row + tile) * (long)n_out : nullptr;
    const float* sc = a.scale ? a.scale + (long)job.slot * n_out : nullptr;
    const float* ft = a.feat_thr ? a.feat_thr + (long)job.slot * n_out : nullptr;
    const bool totals = score && (a.o_tots || a.o_totu || a.o_totconf);
    const int g4 = n_out >> 2;
    const bool vec = (n_out & 3) == 0;
    const bool pow2 = vec && g4 <= 32 && (g4 & (g4 - 1)) == 0;
    // Per-row totals.  pow2: a row's groups of 4 are one aligned segment of a warp, summed by shuffles.  Otherwise each |yhat - y|
    // is parked in the free activation buffer and the row's thread sums them in column order after the barrier: a row's totals do
    // not depend on where in a tile, or in which launch, it lands (a request alone and in a coalesced batch score the same bits).
    float* const dpark = out;
    if (vec) {
      const int limit = nrows * g4;
      const int limit_up = (limit + THREADS - 1) / THREADS * THREADS;
      for (int idx = tid; idx < limit_up; idx += THREADS) {
        const bool live = idx < limit;
        const int r = live ? idx / g4 : 0, j4 = live ? idx - r * g4 : 0;
        float ss = 0.f, su = 0.f;
        if (live) {
          const float4 yh = *reinterpret_cast<const float4*>(in + r * pitch + 4 * j4);
          const long g = (orow + r) * (long)n_out + 4 * j4;
          *reinterpret_cast<float4*>(a.o_model + g) = yh;
          if (score) {
            const float4 yt = __ldg(reinterpret_cast<const float4*>(yg + (long)r * n_out) + j4);
            float4 d;
            d.x = fabsf(yh.x - yt.x); d.y = fabsf(yh.y - yt.y); d.z = fabsf(yh.z - yt.z); d.w = fabsf(yh.w - yt.w);
            if (a.o_tu) *reinterpret_cast<float4*>(a.o_tu + g) = d;
            if (totals && !pow2) *reinterpret_cast<float4*>(dpark + r * pitch + 4 * j4) = d;
            su = d.x * d.x + d.y * d.y + d.z * d.z + d.w * d.w;
            if (sc) {
              const float4 s4 = __ldg(reinterpret_cast<const float4*>(sc) + j4);
              float4 e;
              e.x = d.x * s4.x; e.y = d.y * s4.y; e.z = d.z * s4.z; e.w = d.w * s4.w;
              if (a.o_ts) *reinterpret_cast<float4*>(a.o_ts + g) = e;
              ss = e.x * e.x + e.y * e.y + e.z * e.z + e.w * e.w;
            }
            if (a.o_conf) {
              const float4 t4 = __ldg(reinterpret_cast<const float4*>(ft) + j4);
              float4 c;
              c.x = d.x / t4.x; c.y = d.y / t4.y; c.z = d.z / t4.z; c.w = d.w / t4.w;
              *reinterpret_cast<float4*>(a.o_conf + g) = c;
            }
          }
        }
        if (totals && pow2) {
          for (int o = g4 >> 1; o > 0; o >>= 1) {
            ss += __shfl_xor_sync(0xffffffffu, ss, o);
            su += __shfl_xor_sync(0xffffffffu, su, o);
          }
          if (live && j4 == 0) { rowsum[r] = ss; rowsum[ROWS + r] = su; }
        }
      }
    } else {
      for (int idx = tid; idx < nrows * n_out; idx += THREADS) {
        const int r = idx / n_out, j = idx - r * n_out;
        const float yh = in[r * pitch + j];
        const long g = (orow + r) * (long)n_out + j;
        a.o_model[g] = yh;
        if (score) {
          const float d = fabsf(yh - __ldg(yg + (long)r * n_out + j));
          if (a.o_tu) a.o_tu[g] = d;
          if (sc) {
            const float e = d * __ldg(sc + j);
            if (a.o_ts) a.o_ts[g] = e;
          }
          if (totals) dpark[r * pitch + j] = d;
          if (a.o_conf) a.o_conf[g] = d / __ldg(ft + j);
        }
      }
    }
    __syncthreads();
    if (totals && tid < nrows) {
      const float inv = 1.f / (float)n_out;
      float ss = 0.f, su = 0.f;
      if (pow2) {
        ss = rowsum[tid];
        su = rowsum[ROWS + tid];
      } else {
        const float* dr = dpark + tid * pitch;
        for (int j = 0; j < n_out; ++j) su = fmaf(dr[j], dr[j], su);
        if (sc)
          for (int j = 0; j < n_out; ++j) {
            const float e = dr[j] * __ldg(sc + j);
            ss = fmaf(e, e, ss);
          }
      }
      const float ts = ss * inv, tu = su * inv;
      if (a.o_tots) a.o_tots[orow + tid] = ts;
      if (a.o_totu) a.o_totu[orow + tid] = tu;
      if (a.o_totconf) a.o_totconf[orow + tid] = ts / __ldg(a.agg_thr + job.slot);
    }
    __syncthreads();
  }
}

// The launch plan of an architecture: the largest row tile (128, 64 or 32 rows) whose activation buffers fit next to the weights,
// all layers resident when they fit the budget, else staged layer by layer.  A layer whose whole image does not fit next to even
// the 32-row buffers (a 256 x 256 layer, or 256 x 172 in the feedforward_symmetric default at 172 tags) is staged in blocks of
// output columns.  Fills a.im, a.pitch, a.resident, a.col_block, a.wfloats; returns the row tile and the dynamic shared memory.
int make_plan(const gb_ffnet* net, Args& a, size_t* smem_out) {
  constexpr size_t SMEM_MAX = 227 * 1024;
  a.net = *net;
  a.im = gb::make_ff_image(net, 4);
  int p4 = a.im.max_np / 4 + 1;
  if ((p4 & 1) == 0) ++p4;  // odd number of 16-byte units per row -> conflict-free LDS.128/STS.128
  a.pitch = p4 * 4;
  a.col_block = a.im.max_np;
  int max_layer = 0, max_kp = 0;
  for (int l = 0; l < net->n_layers; ++l) {
    max_layer = max(max_layer, a.im.kp[l] * a.im.np[l] + a.im.np[l]);
    max_kp = max(max_kp, a.im.kp[l]);
  }
  const size_t budget = 220 * 1024;
  int rt = 4;
  size_t smem = 0, act_bytes = 0;
  for (;; rt >>= 1) {  // the largest row tile whose activation buffers fit next to the (resident or per-layer staged) weights
    const int rows = 32 * rt;
    act_bytes = (size_t)(2 * rows * a.pitch + 2 * rows) * sizeof(float);
    a.resident = ((size_t)a.im.total * sizeof(float) + act_bytes) <= budget;
    a.wfloats = gb::round_up(a.resident ? a.im.total : max_layer, 4);
    smem = (size_t)a.wfloats * sizeof(float) + act_bytes;
    if (smem <= SMEM_MAX || rt == 1) break;
  }
  if (smem > SMEM_MAX && act_bytes < SMEM_MAX) {  // column blocks: a multiple of 32 columns (whole warp-task rounds) where possible
    int cb = (int)((SMEM_MAX - act_bytes) / sizeof(float) / (max_kp + 1));
    cb = cb >= 32 ? cb / 32 * 32 : cb / 4 * 4;
    if (cb >= 4) {
      a.col_block = cb;
      int wf = 0;
      for (int l = 0; l < net->n_layers; ++l) {
        const int nb = min(a.im.np[l], cb);
        wf = max(wf, a.im.kp[l] * nb + nb);
      }
      a.wfloats = gb::round_up(wf, 4);
      smem = (size_t)a.wfloats * sizeof(float) + act_bytes;
    }
  }
  GB_REQUIRE(smem <= SMEM_MAX, GB_E_SMEM, "architecture needs %zu bytes of shared memory", smem);
  *smem_out = smem;
  return 32 * rt;
}

}  // namespace

extern "C" int gb_ffae_infer_plan(const gb_ffnet* net, int32_t* rows_per_tile, int32_t* resident) {
  int rc = gb::validate_ffnet(net);
  if (rc != GB_OK) return rc;
  Args a{};
  size_t smem = 0;
  const int rows = make_plan(net, a, &smem);
  if (rows < 0) return rows;
  if (rows_per_tile) *rows_per_tile = rows;
  if (resident) *resident = a.resident;
  return GB_OK;
}

// x_scale == NULL: x is float32.  Otherwise x is float64 and x_scale / x_offset [n_slots][n_in] double are the slot's input scaler.
extern "C" int gb_ffae_infer_score_fma(const gb_ffnet* net, const float* params, const gb_job* jobs, int32_t n_jobs,
                                       int32_t max_rows, const void* x, const double* x_scale, const double* x_offset,
                                       const float* y, const float* scale,
                                       const float* feat_thr, const float* agg_thr, float* out_model,
                                       float* out_tag_scaled, float* out_tag_unscaled, float* out_total_scaled,
                                       float* out_total_unscaled, float* out_conf, float* out_total_conf,
                                       void* stream) {
  Args a{};
  size_t smem = 0;
  const int ROWS = make_plan(net, a, &smem);
  if (ROWS < 0) return ROWS;
  const int rt = ROWS / 32;
  a.n_in = net->dims[0];
  a.n_out = net->dims[net->n_layers];
  a.pstride = (long)gb_ffnet_param_stride(net);
  const bool x64 = x_scale != nullptr;
  a.params = params; a.jobs = jobs; a.y = y; a.scale = scale; a.feat_thr = feat_thr; a.agg_thr = agg_thr;
  a.o_model = out_model; a.o_ts = out_tag_scaled; a.o_tu = out_tag_unscaled; a.o_tots = out_total_scaled;
  a.o_totu = out_total_unscaled; a.o_conf = out_conf; a.o_totconf = out_total_conf;
  if (x64) {
    a.x64 = static_cast<const double*>(x); a.x_scale = x_scale; a.x_offset = x_offset;
  } else {
    a.x = static_cast<const float*>(x);
  }

  int dev = 0, sms = 132;
  GB_CUDA_CHECK(cudaGetDevice(&dev));
  GB_CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const int tiles_per_job = (max_rows + ROWS - 1) / ROWS;
  const int want_chunks = max(1, (4 * sms + n_jobs - 1) / n_jobs);
  int tiles_per_chunk = max(1, tiles_per_job / want_chunks);
  tiles_per_chunk = min(tiles_per_chunk, 16);
  a.rows_per_chunk = tiles_per_chunk * ROWS;
  const int chunks = (tiles_per_job + tiles_per_chunk - 1) / tiles_per_chunk;
  auto launch = [&](auto kern) -> int {
    GB_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    for (int j0 = 0; j0 < n_jobs; j0 += 65535) {  // gridDim.y carries the job index: larger fleets go out as several launches
      a.jobs = jobs + j0;
      kern<<<dim3(chunks, n_jobs - j0 < 65535 ? n_jobs - j0 : 65535), THREADS, smem, (cudaStream_t)stream>>>(a);
    }
    return GB_OK;
  };
  const bool blocked = a.col_block < a.im.max_np;
  int rc;
  if (!x64)
    rc = rt == 4 ? launch(ffae_infer_fma_kernel<4, false, false>) : rt == 2 ? launch(ffae_infer_fma_kernel<2, false, false>)
         : blocked ? launch(ffae_infer_fma_kernel<1, true, false>) : launch(ffae_infer_fma_kernel<1, false, false>);
  else
    rc = rt == 4 ? launch(ffae_infer_fma_kernel<4, false, true>) : rt == 2 ? launch(ffae_infer_fma_kernel<2, false, true>)
         : blocked ? launch(ffae_infer_fma_kernel<1, true, true>) : launch(ffae_infer_fma_kernel<1, false, true>);
  if (rc != GB_OK) return rc;
  GB_CUDA_CHECK(cudaGetLastError());
  return GB_OK;
}
