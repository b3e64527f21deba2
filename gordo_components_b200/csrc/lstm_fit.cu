// K3-fit: training of the stacked-LSTM autoencoders (back-propagation through time), batched over machines.
//
// Replaces KerasLSTMBaseEstimator.fit (gordo/machine/model/models.py:557-616): a primer Adam step on the single window
// X[:L], then `epochs` passes over the lookback windows IN ORDER (shuffle=False, :612-615) in batches of `batch_size`,
// for the stacks of factories/lstm_autoencoder.py:72-103 (every LSTM returns sequences except the last; Dense head;
// MSE or, through gb_lstm_fit_loss, another Keras regression loss; Adam with the Keras defaults).  Windows are never materialised (models.py:713-793): window j of a job is the x rows
// [x_row + j, x_row + j + L) and its target is y row x_row + j + L - 1 + lookahead.
//
// Unlike the Dense autoencoders (one CTA trains one machine with its weights in shared memory), one LSTM stack is
// 1.2 M parameters and 335 MFLOP per window: here one optimizer step of ALL jobs is a sequence of launches whose grids
// span (tile, job) -- the machines are the batch dimension that fills the GPU:
//   forward   t = 0..L-1, layer 0..n-1:  z = [x_t | h_{t-1}] [K; U] + b, gates, (c_t, h_t)   -> saved for the backward pass
//   head      Dense, loss, accuracy, d(loss)/d(yhat), Dense gradients, dh of the last LSTM layer at t = L-1
//   backward  t = L-1..0, layer n-1..0:  gate gradients dz_t (overwrite the saved gates), then
//                                        [dx_t | dh_{t-1}] = dz_t [K; U]^T  (dx_t is the layer below's dh_t)
//   weights   d[K; U] = sum_t [x_t | h_{t-1}]^T dz_t  (one GEMM per layer with reduction length L * batch), db
//   Adam      m += (g-m)(1-b1); v += (g^2-v)(1-b2); w -= lr sqrt(1-b2^t)/(1-b1^t) m/(sqrt(v)+eps)   [3P keras]
// fp32 CUDA cores throughout (a tensor-core path for these GEMMs is the next step for this kernel family).
#include "gb_common.cuh"
#include "lstm_fit_common.cuh"

namespace {

constexpr int MAXB = 32;  // windows per batch handled by one row tile

// ---------------------------------------------------------------------------------------------- forward cell
// grid (ceil(u/16), n_jobs), 256 threads: 16 units x 4 gates = 64 gate columns x up to 32 batch rows.
__global__ void __launch_bounds__(256) lstm_fwd_kernel(const FitArgs a, int l, int t) {
  const gb_job job = a.jobs[blockIdx.y];
  const int nb = job_batch(job, a.step[0], a.step[1]);
  if (nb == 0) return;
  const Lay ly = a.lay[l];
  const int u = ly.u, in = ly.in, KK = in + u, u4 = 4 * u;
  const int u0 = blockIdx.x * 16;
  float* ws = a.ws + (long)blockIdx.y * a.ws_stride;
  const float* P = a.params + (long)job.slot * a.pstride + ly.kofs;  // [K; U] rows, then bias
  __shared__ float sA[MAXB][33];
  __shared__ float sW[32][65];
  __shared__ float sZ[MAXB][65];
  const int tid = threadIdx.x, col = tid & 63, rg = tid >> 6;  // thread: gate column `col`, rows rg, rg+4, ...
  const int gate = col >> 4, unit = u0 + (col & 15);
  const bool ucol = unit < u;
  const int pcol = gate * u + (ucol ? unit : 0);
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
  const float* hprev = ws + ly.hofs + (long)(t - 1) * MAXB * u;
  const float* below = l > 0 ? ws + a.lay[l - 1].hofs + (long)t * MAXB * a.lay[l - 1].u : nullptr;
  for (int k0 = 0; k0 < KK; k0 += 32) {
    // A tile: rows b < nb, columns k0 .. k0+31 of [input_t | h_{t-1}]
    for (int i = tid; i < MAXB * 32; i += 256) {
      const int b = i >> 5, k = k0 + (i & 31);
      float v = 0.f;
      if (b < nb && k < KK) {
        if (k < in) v = l == 0 ? __ldg(a.x + (job.x_row + a.step[0] + b + t) * (long)a.F + k) : below[b * in + k];
        else v = t > 0 ? hprev[b * u + (k - in)] : 0.f;
      }
      sA[b][i & 31] = v;
    }
    for (int i = tid; i < 32 * 64; i += 256) {
      const int kk = i >> 6, c = i & 63, k = k0 + kk;
      const int g = c >> 4, un = u0 + (c & 15);
      sW[kk][c] = (k < KK && un < u) ? __ldg(P + (long)k * u4 + g * u + un) : 0.f;
    }
    __syncthreads();
#pragma unroll 8
    for (int kk = 0; kk < 32; ++kk) {
      const float w = sW[kk][col];
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = fmaf(sA[rg + 4 * i][kk], w, acc[i]);
    }
    __syncthreads();
  }
  const float bias = ucol ? __ldg(P + (long)KK * u4 + pcol) : 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) sZ[rg + 4 * i][col] = acc[i] + bias;
  __syncthreads();
  // cell update: (row, unit) pairs
  float* Z = ws + ly.zofs + (long)t * MAXB * u4;
  float* C = ws + ly.cofs + (long)t * MAXB * u;
  float* H = ws + ly.hofs + (long)t * MAXB * u;
  const float* Cp = ws + ly.cofs + (long)(t - 1) * MAXB * u;
  for (int i = tid; i < MAXB * 16; i += 256) {
    const int b = i >> 4, uu = i & 15, un = u0 + uu;
    if (b < nb && un < u) {
      const float ig = sigm(sZ[b][uu]), fg = sigm(sZ[b][16 + uu]), gg = gb::apply_act(ly.act, sZ[b][32 + uu]), og = sigm(sZ[b][48 + uu]);
      const float cp = t > 0 ? Cp[b * u + un] : 0.f;
      const float c = fmaf(fg, cp, ig * gg);
      Z[b * u4 + un] = ig; Z[b * u4 + u + un] = fg; Z[b * u4 + 2 * u + un] = gg; Z[b * u4 + 3 * u + un] = og;
      C[b * u + un] = c;
      H[b * u + un] = og * gb::apply_act(ly.act, c);
    }
  }
}

// ---------------------------------------------------------------------------------------------- Dense head, loss, its gradients
// grid n_jobs, 256 threads.  Dynamic smem: h [B][u], dout [B][T_out], yhat [B][T_out].
__global__ void __launch_bounds__(256) lstm_head_kernel(const FitArgs a) {
  const gb_job job = a.jobs[blockIdx.x];
  const int nb = job_batch(job, a.step[0], a.step[1]);
  if (nb == 0) return;
  extern __shared__ float sm[];
  const Lay top = a.lay[a.n_layers - 1];
  const int u = top.u, T = a.T_out;
  float* sh = sm;
  float* sd = sh + MAXB * u;
  float* sy = sd + MAXB * T;
  __shared__ float red[256];
  float* ws = a.ws + (long)blockIdx.x * a.ws_stride;
  const float* P = a.params + (long)job.slot * a.pstride + a.dofs;  // Wd [u][T], bd [T]
  float* G = ws + a.gofs + a.dofs;
  const float* H = ws + top.hofs + (long)(a.L - 1) * MAXB * u;
  const int tid = threadIdx.x;
  for (int i = tid; i < nb * u; i += 256) sh[i] = H[i];
  __syncthreads();
  const float inv = 2.0f / (float)(nb * T);
  const float linv = 1.0f / (float)(nb * T);
  float lsum = 0.f;
  for (int i = tid; i < nb * T; i += 256) {
    const int b = i / T, o = i - b * T;
    float z = __ldg(P + (long)u * T + o);
    for (int k = 0; k < u; ++k) z = fmaf(sh[b * u + k], __ldg(P + (long)k * T + o), z);
    const float yh = gb::apply_act(a.out_act, z);
    const float tgt = __ldg(a.y + (job.x_row + a.step[0] + b + a.L - 1 + a.lookahead) * (long)T + o);
    sy[i] = yh;
    if (a.loss == GB_LOSS_MSE) {  // the MSE arithmetic of gb_lstm_fit, unchanged
      const float d = yh - tgt;
      lsum += d * d;
      sd[i] = inv * d * gb::act_grad_from_output(a.out_act, yh);
    } else {
      lsum += gb::loss_value(a.loss, yh, tgt);
      sd[i] = linv * gb::loss_grad(a.loss, yh, tgt) * gb::act_grad_from_output(a.out_act, yh);
    }
  }
  red[tid] = lsum;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (tid < s) red[tid] += red[tid + s];
    __syncthreads();
  }
  if (tid == 0) a.loss_sum[blockIdx.x] += red[0] / (float)(nb * T) * (float)nb;
  // accuracy (metrics=["accuracy"] on 2-D float targets: argmax match; width 1: thresholded match)
  if (tid < nb) {
    const float* tg = a.y + (job.x_row + a.step[0] + tid + a.L - 1 + a.lookahead) * (long)T;
    float hit;
    if (T == 1) {
      hit = ((sy[tid] > 0.5f ? 1.f : 0.f) == __ldg(tg)) ? 1.f : 0.f;
    } else {
      int am = 0, at = 0;
      for (int o = 1; o < T; ++o) {
        if (sy[tid * T + o] > sy[tid * T + am]) am = o;
        if (__ldg(tg + o) > __ldg(tg + at)) at = o;
      }
      hit = am == at ? 1.f : 0.f;
    }
    atomicAdd(a.hit_sum + blockIdx.x, hit);
  }
  // dWd[k][o] = sum_b h[b][k] dout[b][o];  dbd[o] = sum_b dout[b][o]
  for (int i = tid; i < u * T; i += 256) {
    const int k = i / T, o = i - k * T;
    float g = 0.f;
    for (int b = 0; b < nb; ++b) g = fmaf(sh[b * u + k], sd[b * T + o], g);
    G[i] = g;
  }
  for (int o = tid; o < T; o += 256) {
    float g = 0.f;
    for (int b = 0; b < nb; ++b) g += sd[b * T + o];
    G[(long)u * T + o] = g;
  }
  // dh of the last LSTM layer at t = L-1: dh[b][k] = sum_o dout[b][o] Wd[k][o]
  float* DH = ws + a.topdh;
  for (int i = tid; i < nb * u; i += 256) {
    const int b = i / u, k = i - b * u;
    float g = 0.f;
    for (int o = 0; o < T; ++o) g = fmaf(sd[b * T + o], __ldg(P + (long)k * T + o), g);
    DH[i] = g;
  }
}

// ---------------------------------------------------------------------------------------------- backward: [dx_t | dh_{t-1}] = dz_t [K; U]^T
// grid (ceil(cols/64), n_jobs) over the columns that are needed (layer 0 has no dx), 256 threads.
__global__ void __launch_bounds__(256) lstm_bwd_input_kernel(const FitArgs a, int l, int t) {
  const gb_job job = a.jobs[blockIdx.y];
  const int nb = job_batch(job, a.step[0], a.step[1]);
  if (nb == 0) return;
  const Lay ly = a.lay[l];
  const int u = ly.u, in = ly.in, KK = in + u, u4 = 4 * u;
  const int kbase = (l == 0 ? in : 0) + blockIdx.x * 64;  // first output column (row of [K; U]) of this CTA
  float* ws = a.ws + (long)blockIdx.y * a.ws_stride;
  const float* P = a.params + (long)job.slot * a.pstride + ly.kofs;
  const float* Z = ws + ly.zofs + (long)t * MAXB * u4;
  __shared__ float sA[MAXB][33];
  __shared__ float sW[64][33];
  const int tid = threadIdx.x, col = tid & 63, rg = tid >> 6;
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
  for (int c0 = 0; c0 < u4; c0 += 32) {
    for (int i = tid; i < MAXB * 32; i += 256) {
      const int b = i >> 5, c = c0 + (i & 31);
      sA[b][i & 31] = (b < nb && c < u4) ? Z[(long)b * u4 + c] : 0.f;
    }
    for (int i = tid; i < 64 * 32; i += 256) {
      const int kk = i >> 5, c = c0 + (i & 31), k = kbase + kk;
      sW[kk][i & 31] = (k < KK && c < u4) ? __ldg(P + (long)k * u4 + c) : 0.f;
    }
    __syncthreads();
#pragma unroll 8
    for (int cc = 0; cc < 32; ++cc) {
      const float w = sW[col][cc];
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = fmaf(sA[rg + 4 * i][cc], w, acc[i]);
    }
    __syncthreads();
  }
  const int k = kbase + col;
  if (k >= KK) return;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int b = rg + 4 * i;
    if (b >= nb) continue;
    if (k < in) ws[a.lay[l - 1].dhofs + (long)t * MAXB * in + b * in + k] = acc[i];  // the layer below's dh at time t (its width = our input width)
    else ws[ly.nxofs + b * u + (k - in)] = acc[i];                                     // dh_next of this layer
  }
}

// ---------------------------------------------------------------------------------------------- weight gradients
// d[K; U][k][c] = sum_{t,b} [x_t | h_{t-1}][b][k] dz_t[b][c];  db[c] = sum_{t,b} dz_t[b][c]
// grid (ceil(4u/64), ceil((in+u)/32), n_jobs), 256 threads: tile of 32 rows k x 64 columns c, reduction over (t, b).
__global__ void __launch_bounds__(256) lstm_wgrad_kernel(const FitArgs a, int l) {
  const gb_job job = a.jobs[blockIdx.z];
  const int nb = job_batch(job, a.step[0], a.step[1]);
  if (nb == 0) return;
  const Lay ly = a.lay[l];
  const int u = ly.u, in = ly.in, KK = in + u, u4 = 4 * u;
  const int c0 = blockIdx.x * 64, k0 = blockIdx.y * 32;
  float* ws = a.ws + (long)blockIdx.z * a.ws_stride;
  float* G = ws + a.gofs + ly.kofs;
  __shared__ float sA[MAXB][33];  // [b][k]
  __shared__ float sZ[MAXB][65];  // [b][c]
  const int tid = threadIdx.x, col = tid & 63, rg = tid >> 6;  // thread: column c0+col, rows k0 + rg + 4 i
  float acc[8], bsum = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
  for (int t = 0; t < a.L; ++t) {
    const float* Z = ws + ly.zofs + (long)t * MAXB * u4;
    const float* below = l > 0 ? ws + a.lay[l - 1].hofs + (long)t * MAXB * in : nullptr;
    const float* hprev = ws + ly.hofs + (long)(t - 1) * MAXB * u;
    for (int i = tid; i < MAXB * 32; i += 256) {
      const int b = i >> 5, k = k0 + (i & 31);
      float v = 0.f;
      if (b < nb && k < KK) {
        if (k < in) v = l == 0 ? __ldg(a.x + (job.x_row + a.step[0] + b + t) * (long)a.F + k) : below[b * in + k];
        else v = t > 0 ? hprev[b * u + (k - in)] : 0.f;
      }
      sA[b][i & 31] = v;
    }
    for (int i = tid; i < MAXB * 64; i += 256) {
      const int b = i >> 6, c = c0 + (i & 63);
      sZ[b][i & 63] = (b < nb && c < u4) ? Z[(long)b * u4 + c] : 0.f;
    }
    __syncthreads();
#pragma unroll 4
    for (int b = 0; b < MAXB; ++b) {
      const float z = sZ[b][col];
      if (rg == 0) bsum += z;
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = fmaf(sA[b][rg + 4 * i], z, acc[i]);
    }
    __syncthreads();
  }
  const int c = c0 + col;
  if (c >= u4) return;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int k = k0 + rg + 4 * i;
    if (k < KK) G[(long)k * u4 + c] = acc[i];
  }
  if (blockIdx.y == 0 && rg == 0) G[(long)KK * u4 + c] = bsum;
}

// ---------------------------------------------------------------------------------------------- orthogonal initialiser
// Keras' Orthogonal for a recurrent kernel [u, 4u] [3P]: QR of a [4u, u] standard-normal draw, Q's columns sign-corrected so that
// diag(R) > 0, transposed.  That Q is what Gram-Schmidt gives, so: one CTA per matrix orthonormalises the rows of its own
// [rows, cols] normal draw `g` in place (float64, modified Gram-Schmidt) and writes them rounded to float32.
__global__ void __launch_bounds__(256) orthonormal_rows_kernel(double* g, int rows, int cols, float* out, long out_stride) {
  __shared__ double s_red[8];
  double* a = g + (long)blockIdx.x * rows * cols;
  float* o = out + (long)blockIdx.x * out_stride;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int i = 0; i < rows; ++i) {
    double* ri = a + (long)i * cols;
    double s = 0.;
    for (int c = threadIdx.x; c < cols; c += 256) s += ri[c] * ri[c];
    for (int k = 16; k > 0; k >>= 1) s += __shfl_xor_sync(0xffffffffu, s, k);
    if (lane == 0) s_red[warp] = s;
    __syncthreads();
    double norm2 = 0.;
#pragma unroll
    for (int w = 0; w < 8; ++w) norm2 += s_red[w];
    const double inv = 1. / sqrt(norm2);
    for (int c = threadIdx.x; c < cols; c += 256) {
      const double v = ri[c] * inv;
      ri[c] = v;
      o[(long)i * cols + c] = (float)v;
    }
    __syncthreads();
    for (int j = i + 1 + warp; j < rows; j += 8) {  // take row i out of every later row: one warp per row
      double* rj = a + (long)j * cols;
      double d = 0.;
      for (int c = lane; c < cols; c += 32) d += rj[c] * ri[c];
      for (int k = 16; k > 0; k >>= 1) d += __shfl_xor_sync(0xffffffffu, d, k);
      for (int c = lane; c < cols; c += 32) rj[c] -= d * ri[c];
    }
    __syncthreads();
  }
}

// fit_driver's policy for this family: one MAXB-row tile per batch, the head of a job in one CTA
struct Fp32Fit {
  static constexpr int max_batch = MAXB;
  static constexpr const char* who = "this kernel family";
  static constexpr int head_rows = 0;
  static int rows(int) { return MAXB; }
  size_t head_smem = 0;

  int prepare(const FitArgs& a) {
    head_smem = (size_t)(MAXB * a.lay[a.n_layers - 1].u + 2 * MAXB * a.T_out) * sizeof(float);
    GB_REQUIRE(head_smem <= 200 * 1024, GB_E_SMEM, "Dense head needs %zu bytes of shared memory", head_smem);
    GB_CUDA_CHECK(cudaFuncSetAttribute(lstm_head_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)head_smem));
    return GB_OK;
  }

  void record(const FitArgs& a, int n_jobs, cudaStream_t st) const {
    for (int t = 0; t < a.L; ++t)
      for (int l = 0; l < a.n_layers; ++l) lstm_fwd_kernel<<<dim3((a.lay[l].u + 15) / 16, n_jobs), 256, 0, st>>>(a, l, t);
    lstm_head_kernel<<<n_jobs, 256, head_smem, st>>>(a);
    for (int t = a.L - 1; t >= 0; --t)
      for (int l = a.n_layers - 1; l >= 0; --l) {
        const Lay& ly = a.lay[l];
        lstm_bwd_gates_kernel<<<dim3((MAXB * ly.u + 255) / 256, n_jobs), 256, 0, st>>>(a, l, t);
        const int cols = l == 0 ? ly.u : ly.in + ly.u;
        if (t > 0 || l > 0) lstm_bwd_input_kernel<<<dim3((cols + 63) / 64, n_jobs), 256, 0, st>>>(a, l, t);
      }
    for (int l = 0; l < a.n_layers; ++l) {
      const Lay& ly = a.lay[l];
      lstm_wgrad_kernel<<<dim3((4 * ly.u + 63) / 64, (ly.in + ly.u + 31) / 32, n_jobs), 256, 0, st>>>(a, l);
    }
  }
};

}  // namespace

extern "C" {

size_t gb_lstm_fit_workspace_bytes(const gb_lstmnet* net, int32_t n_jobs) {
  if (gb::validate_lstmnet(net) != GB_OK || n_jobs < 0) return 0;
  FitArgs a{};
  return workspace_bytes(layout(net, MAXB, 0, &a), n_jobs);
}

int gb_lstm_fit(const gb_lstmnet* net, float* params, float* adam_m, float* adam_v, int32_t* adam_t, const gb_job* jobs, int32_t n_jobs,
                int32_t max_windows, const float* x, const float* y, const gb_lstm_fit_hparams* hp, void* workspace, float* out_loss,
                float* out_acc, void* stream) {
  return gb_lstm_fit_loss(net, params, adam_m, adam_v, adam_t, jobs, n_jobs, max_windows, x, y, hp, workspace, out_loss, out_acc,
                          GB_LOSS_MSE, stream);
}

int gb_lstm_fit_loss(const gb_lstmnet* net, float* params, float* adam_m, float* adam_v, int32_t* adam_t, const gb_job* jobs,
                     int32_t n_jobs, int32_t max_windows, const float* x, const float* y, const gb_lstm_fit_hparams* hp, void* workspace,
                     float* out_loss, float* out_acc, int32_t loss, void* stream) {
  return gb_lstm_fit_opt(net, params, adam_m, adam_v, adam_t, jobs, n_jobs, max_windows, x, y, hp, workspace, out_loss, out_acc, loss,
                         nullptr, stream);
}

int gb_lstm_fit_opt(const gb_lstmnet* net, float* params, float* adam_m, float* adam_v, int32_t* adam_t, const gb_job* jobs,
                    int32_t n_jobs, int32_t max_windows, const float* x, const float* y, const gb_lstm_fit_hparams* hp, void* workspace,
                    float* out_loss, float* out_acc, int32_t loss, const gb_optimizer* opt, void* stream) {
  return fit_driver(Fp32Fit{}, net, params, adam_m, adam_v, adam_t, jobs, n_jobs, max_windows, x, y, hp, workspace, out_loss, out_acc,
                    loss, opt, nullptr, nullptr, nullptr, nullptr, stream);
}

int gb_lstm_fit_stop(const gb_lstmnet* net, float* params, float* adam_m, float* adam_v, int32_t* adam_t, const gb_job* jobs,
                     int32_t n_jobs, int32_t max_windows, const float* x, const float* y, const gb_lstm_fit_hparams* hp, void* workspace,
                     float* out_loss, float* out_acc, int32_t loss, const gb_optimizer* opt, const gb_fit_stop* stop, float* best_params,
                     int32_t* out_epochs, int32_t* out_best_epoch, void* stream) {
  return fit_driver(Fp32Fit{}, net, params, adam_m, adam_v, adam_t, jobs, n_jobs, max_windows, x, y, hp, workspace, out_loss, out_acc,
                    loss, opt, stop, best_params, out_epochs, out_best_epoch, stream);
}

size_t gb_lstm_fit_stop_state_bytes(int32_t n_jobs) { return n_jobs < 0 ? 0 : lstm_stop::state_bytes(n_jobs); }

int gb_orthonormal_rows(double* g, int32_t n_mats, int32_t rows, int32_t cols, float* out, int64_t out_offset, int64_t out_stride,
                        void* stream) {
  GB_REQUIRE(g && out, GB_E_ARG, "g/out must be non-NULL");
  GB_REQUIRE(n_mats >= 0 && rows >= 1 && cols >= rows, GB_E_SHAPE, "rows=%d cols=%d: need 1 <= rows <= cols", rows, cols);
  GB_REQUIRE(out_offset >= 0 && out_stride >= (int64_t)rows * cols, GB_E_ARG, "out_stride=%lld is shorter than one matrix", (long long)out_stride);
  if (n_mats == 0) return GB_OK;
  orthonormal_rows_kernel<<<n_mats, 256, 0, (cudaStream_t)stream>>>(g, rows, cols, out + out_offset, out_stride);
  GB_CUDA_CHECK(cudaGetLastError());
  return GB_OK;
}

}  // extern "C"
