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
#include "lstm_fit_stop.cuh"

namespace {

constexpr int MAXB = 32;  // windows per batch handled by one row tile
constexpr int LSTM_MAX_UNITS = 512;
constexpr int LSTM_MAX_FEATURES = 512;

struct Lay {
  int in, u;       // input width, units
  int act;
  long kofs;       // offset of [K; U] (rows in + u, 4u columns) in the parameter vector; bias follows
  long zofs, cofs, hofs, dhofs, nxofs;  // workspace offsets (floats, per job): gates [L][B][4u], c / h [L][B][u], dh_seq [L][B][u], (dh_next, dc_next) [2][B][u]
};

struct FitArgs {
  int n_layers, L, F, T_out, out_act, lookahead;
  Lay lay[GB_MAX_LAYERS];
  long dofs;        // Dense kernel offset in the parameter vector
  long pstride, ws_stride;  // floats per slot / per job
  long gofs;        // gradient vector offset in the job workspace
  long topdh;       // [B][u_top] dh of the last LSTM layer at t = L-1
  float* params;
  float *adam_m, *adam_v;
  int* adam_t;
  const gb_job* jobs;
  const float *x, *y;
  float* ws;
  float *loss_sum, *hit_sum;  // [n_jobs]
  const int* step;            // device: {first window, nominal batch size} of the optimizer step being replayed (the launch
                              // sequence of one step is captured once as a CUDA graph; only these two numbers change)
  float lr, b1, b2, eps;
  int loss;                   // gb_loss of the head
  gb_optimizer opt;            // gb_lstm_fit_opt with another optimizer than plain Adam (lstm_opt_kernel)
};

__device__ __forceinline__ float sigm(float z) { return 1.f / (1.f + expf(-z)); }
__device__ __forceinline__ int job_batch(const gb_job& job, int win0, int bsz) { return max(0, min(bsz, job.n_rows - win0)); }

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

// ---------------------------------------------------------------------------------------------- backward: gate gradients
// grid (ceil(MAXB*u/256), n_jobs).  Overwrites the saved gates of (l, t) with dz, updates dc_next.
__global__ void __launch_bounds__(256) lstm_bwd_gates_kernel(const FitArgs a, int l, int t) {
  const gb_job job = a.jobs[blockIdx.y];
  const int nb = job_batch(job, a.step[0], a.step[1]);
  if (nb == 0) return;
  const Lay ly = a.lay[l];
  const int u = ly.u, u4 = 4 * u;
  const int i = blockIdx.x * 256 + threadIdx.x;
  const int b = i / u, un = i - b * u;
  if (b >= nb) return;
  float* ws = a.ws + (long)blockIdx.y * a.ws_stride;
  float* Z = ws + ly.zofs + (long)t * MAXB * u4 + (long)b * u4;
  const float ig = Z[un], fg = Z[u + un], gg = Z[2 * u + un], og = Z[3 * u + un];
  const float c = ws[ly.cofs + (long)t * MAXB * u + b * u + un];
  const float cp = t > 0 ? ws[ly.cofs + (long)(t - 1) * MAXB * u + b * u + un] : 0.f;
  float* nx = ws + ly.nxofs;  // dh_next [B][u], dc_next [B][u]
  const bool last_t = t == a.L - 1;
  float dh = last_t ? 0.f : nx[b * u + un];
  if (l == a.n_layers - 1) {
    if (last_t) dh += ws[a.topdh + b * u + un];
  } else {
    dh += ws[ly.dhofs + (long)t * MAXB * u + b * u + un];
  }
  const float ac = gb::apply_act(ly.act, c);
  const float dc = dh * og * gb::act_grad_from_output(ly.act, ac) + (last_t ? 0.f : nx[MAXB * u + b * u + un]);
  Z[un] = dc * gg * ig * (1.f - ig);
  Z[u + un] = dc * cp * fg * (1.f - fg);
  Z[2 * u + un] = dc * ig * gb::act_grad_from_output(ly.act, gg);
  Z[3 * u + un] = dh * ac * og * (1.f - og);
  nx[MAXB * u + b * u + un] = dc * fg;
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

// ---------------------------------------------------------------------------------------------- Adam
__global__ void __launch_bounds__(256) lstm_adam_kernel(const FitArgs a, long n_params) {
  const gb_job job = a.jobs[blockIdx.y];
  if (job_batch(job, a.step[0], a.step[1]) == 0) return;
  const int t = a.adam_t[job.slot] + 1;
  const float alpha = (float)((double)a.lr * sqrt(1.0 - pow((double)a.b2, (double)t)) / (1.0 - pow((double)a.b1, (double)t)));
  const float* G = a.ws + (long)blockIdx.y * a.ws_stride + a.gofs;
  float* P = a.params + (long)job.slot * a.pstride;
  float* M = a.adam_m + (long)job.slot * a.pstride;
  float* V = a.adam_v + (long)job.slot * a.pstride;
  for (long i = (long)blockIdx.x * 256 + threadIdx.x; i < n_params; i += (long)gridDim.x * 256) {
    const float g = G[i];
    const float m = M[i] + (g - M[i]) * (1.f - a.b1);
    const float v = V[i] + (g * g - V[i]) * (1.f - a.b2);
    M[i] = m;
    V[i] = v;
    P[i] -= alpha * m / (sqrtf(v) + a.eps);
  }
}
// Every other optimizer than plain Adam (gb::opt_update; state slots 0 / 1 = adam_m / adam_v), captured in place of lstm_adam_kernel.
// The per-step scalars come from the slot's step count, once per CTA (for Nadam a product over the slot's steps, a few cycles each).
__global__ void __launch_bounds__(256) lstm_opt_kernel(const FitArgs a, long n_params) {
  const gb_job job = a.jobs[blockIdx.y];
  if (job_batch(job, a.step[0], a.step[1]) == 0) return;
  __shared__ gb::OptStep s_st;
  if (threadIdx.x == 0) s_st = gb::opt_step_at(a.opt, a.adam_t[job.slot] + 1);
  __syncthreads();
  const gb::OptStep st = s_st;
  const float* G = a.ws + (long)blockIdx.y * a.ws_stride + a.gofs;
  float* P = a.params + (long)job.slot * a.pstride;
  float* S0 = a.adam_m + (long)job.slot * a.pstride;
  float* S1 = a.adam_v + (long)job.slot * a.pstride;
  for (long i = (long)blockIdx.x * 256 + threadIdx.x; i < n_params; i += (long)gridDim.x * 256) {
    float w = P[i], s0 = S0[i], s1 = S1[i];
    gb::opt_update(a.opt, st, w, G[i], s0, s1);
    P[i] = w;
    S0[i] = s0;
    S1[i] = s1;
  }
}
__global__ void lstm_bump_kernel(const FitArgs a, int n_jobs) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n_jobs && job_batch(a.jobs[j], a.step[0], a.step[1]) > 0) a.adam_t[a.jobs[j].slot] += 1;
}
__global__ void lstm_set_step_kernel(int* step, int win0, int bsz) {
  step[0] = win0;
  step[1] = bsz;
}
// epoch bookkeeping: history[job][epoch] = sums / n_windows; sums reset
__global__ void lstm_epoch_kernel(const gb_job* jobs, int n_jobs, float* loss_sum, float* hit_sum, float* out_loss, float* out_acc, int epoch, int epochs) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n_jobs) return;
  if (epoch >= 0) {
    const float n = (float)max(jobs[j].n_rows, 1);
    out_loss[(long)j * epochs + epoch] = loss_sum[j] / n;
    out_acc[(long)j * epochs + epoch] = hit_sum[j] / n;
  }
  loss_sum[j] = 0.f;
  hit_sum[j] = 0.f;
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

int validate(const gb_lstmnet* net) {
  GB_REQUIRE(net != nullptr, GB_E_ARG, "net is NULL");
  GB_REQUIRE(net->n_layers >= 1 && net->n_layers <= GB_MAX_LAYERS, GB_E_SHAPE, "n_layers=%d outside [1,%d]", net->n_layers, GB_MAX_LAYERS);
  GB_REQUIRE(net->n_features >= 1 && net->n_features <= LSTM_MAX_FEATURES && net->n_features_out >= 1 && net->n_features_out <= LSTM_MAX_FEATURES,
             GB_E_SHAPE, "n_features/n_features_out outside [1,%d]", LSTM_MAX_FEATURES);
  GB_REQUIRE(net->lookback >= 1, GB_E_ARG, "lookback=%d must be >= 1", net->lookback);
  for (int l = 0; l < net->n_layers; ++l) {
    GB_REQUIRE(net->units[l] >= 1 && net->units[l] <= LSTM_MAX_UNITS, GB_E_SHAPE, "units[%d]=%d outside [1,%d]", l, net->units[l], LSTM_MAX_UNITS);
    GB_REQUIRE(net->act[l] >= GB_ACT_LINEAR && net->act[l] <= GB_ACT_SIGMOID, GB_E_ARG, "act[%d] unknown", l);
  }
  return GB_OK;
}

// workspace layout of one job (floats); returns the total
long layout(const gb_lstmnet* net, FitArgs* a) {
  long ofs = 0, pofs = 0;
  int in = net->n_features;
  const long L = net->lookback;
  for (int l = 0; l < net->n_layers; ++l) {
    const int u = net->units[l];
    Lay& ly = a->lay[l];
    ly.in = in; ly.u = u; ly.act = net->act[l];
    ly.kofs = pofs;
    pofs += 4L * u * (in + u + 1);
    ly.zofs = ofs; ofs += L * MAXB * 4 * u;
    ly.cofs = ofs; ofs += L * MAXB * u;
    ly.hofs = ofs; ofs += L * MAXB * u;
    ly.dhofs = ofs; ofs += (l + 1 < net->n_layers) ? L * MAXB * u : 0;
    ly.nxofs = ofs; ofs += 2L * MAXB * u;
    in = u;
  }
  a->dofs = pofs;
  a->topdh = ofs; ofs += (long)MAXB * in;
  a->gofs = ofs; ofs += (long)gb_lstm_param_stride(net);
  return (ofs + 3) / 4 * 4;
}

}  // namespace

extern "C" {

size_t gb_lstm_fit_workspace_bytes(const gb_lstmnet* net, int32_t n_jobs) {
  if (validate(net) != GB_OK || n_jobs < 0) return 0;
  FitArgs a{};
  return (size_t)(layout(net, &a) * (long)n_jobs + 2L * n_jobs + 4) * sizeof(float);
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

// gb_lstm_fit_opt (stop NULL: the step graph and launches as they have always been) and gb_lstm_fit_stop
static int launch_fit(const gb_lstmnet* net, float* params, float* adam_m, float* adam_v, int32_t* adam_t, const gb_job* jobs,
                      int32_t n_jobs, int32_t max_windows, const float* x, const float* y, const gb_lstm_fit_hparams* hp, void* workspace,
                      float* out_loss, float* out_acc, int32_t loss, const gb_optimizer* opt, const gb_fit_stop* stop, float* best_params,
                      int32_t* out_epochs, int32_t* out_best_epoch, void* stream) {
  int rc = validate(net);
  if (rc != GB_OK) return rc;
  if ((rc = gb::validate_optimizer(opt)) != GB_OK) return rc;
  GB_REQUIRE(loss >= GB_LOSS_MSE && loss <= GB_LOSS_LOG_COSH, GB_E_ARG, "loss=%d unknown (gb_loss: 0..5)", loss);
  GB_REQUIRE(params && adam_m && adam_v && adam_t && jobs && x && y && hp && workspace && out_loss && out_acc, GB_E_ARG, "NULL argument");
  GB_REQUIRE(n_jobs >= 0 && n_jobs <= 65535 && max_windows >= 0, GB_E_ARG, "bad n_jobs/max_windows");
  GB_REQUIRE(hp->epochs >= 0 && hp->batch_size >= 1, GB_E_ARG, "epochs=%d batch_size=%d", hp->epochs, hp->batch_size);
  GB_REQUIRE(hp->batch_size <= MAXB, GB_E_SHAPE, "batch_size=%d: this kernel family handles batches of at most %d windows", hp->batch_size, MAXB);
  GB_REQUIRE(hp->lookahead >= 0, GB_E_ARG, "Value of `lookahead` can not be negative, is %d", hp->lookahead);
  if (stop != nullptr) {
    GB_REQUIRE(best_params && out_epochs && out_best_epoch, GB_E_ARG, "stop needs best_params, out_epochs and out_best_epoch");
    GB_REQUIRE(gb::aligned16(best_params), GB_E_ARG, "best_params must be 16-byte aligned");
    if ((rc = lstm_stop::validate(stop, n_jobs)) != GB_OK) return rc;
  }
  if (n_jobs == 0) return GB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  FitArgs a{};
  a.n_layers = net->n_layers; a.L = net->lookback; a.F = net->n_features; a.T_out = net->n_features_out; a.out_act = net->out_act;
  a.lookahead = hp->lookahead;
  a.ws_stride = layout(net, &a);
  a.pstride = (long)gb_lstm_param_stride(net);
  a.params = params; a.adam_m = adam_m; a.adam_v = adam_v; a.adam_t = adam_t; a.jobs = jobs; a.x = x; a.y = y;
  a.ws = static_cast<float*>(workspace);
  a.loss_sum = a.ws + a.ws_stride * n_jobs;
  a.hit_sum = a.loss_sum + n_jobs;
  a.lr = hp->lr; a.b1 = hp->beta1; a.b2 = hp->beta2; a.eps = hp->eps;
  const bool use_opt = !gb::plain_adam(opt);
  if (opt != nullptr && !use_opt) { a.lr = opt->lr; a.b1 = opt->beta1; a.b2 = opt->beta2; a.eps = opt->eps; }  // plain Adam: the Adam kernel
  if (use_opt) a.opt = *opt;
  a.loss = loss;
  const long n_params = (long)gb_lstm_param_count(net);
  const int u_top = net->units[net->n_layers - 1];
  const size_t head_smem = (size_t)(MAXB * u_top + 2 * MAXB * net->n_features_out) * sizeof(float);
  GB_REQUIRE(head_smem <= 200 * 1024, GB_E_SMEM, "Dense head needs %zu bytes of shared memory", head_smem);
  GB_CUDA_CHECK(cudaFuncSetAttribute(lstm_head_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)head_smem));
  const int jb = (n_jobs + 127) / 128;

  int* d_step = reinterpret_cast<int*>(a.hit_sum + n_jobs);
  a.step = d_step;
  const lstm_stop::Run run(workspace, gb_lstm_fit_workspace_bytes(net, n_jobs), jobs, n_jobs, hp->epochs, out_epochs, out_best_epoch,
                           params, best_params, a.pstride, n_params);
  if (stop != nullptr) {
    run.init(stop, st);
    a.jobs = run.job_copy;  // a job that stops gets n_rows 0 here, so job_batch gives it no windows
  }
  // One optimizer step is ~2 600 small launches (18 per timestep): captured once as a CUDA graph and replayed per step, the
  // step's (first window, batch size) being read from device memory -- launch overhead was >90 % of a step for few machines.
  cudaGraphExec_t gexec = nullptr;
  rc = capture_step(&gexec, stop != nullptr ? run.live : nullptr, [&](cudaStream_t st) {
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
    if (use_opt)
      lstm_opt_kernel<<<dim3((unsigned)((n_params + 256 * 8 - 1) / (256 * 8)), n_jobs), 256, 0, st>>>(a, n_params);
    else
      lstm_adam_kernel<<<dim3((unsigned)((n_params + 256 * 8 - 1) / (256 * 8)), n_jobs), 256, 0, st>>>(a, n_params);
    lstm_bump_kernel<<<jb, 128, 0, st>>>(a, n_jobs);
  });
  if (rc != GB_OK) return rc;
  auto step = [&](int win0, int bsz) -> int {
    lstm_set_step_kernel<<<1, 1, 0, st>>>(d_step, win0, bsz);
    const cudaError_t ce = cudaGraphLaunch(gexec, st);
    if (ce != cudaSuccess) {
      gb::set_error("cudaGraphLaunch failed: %s", cudaGetErrorString(ce));
      return GB_E_CUDA;
    }
    return GB_OK;
  };

  lstm_epoch_kernel<<<jb, 128, 0, st>>>(jobs, n_jobs, a.loss_sum, a.hit_sum, out_loss, out_acc, -1, hp->epochs);
  if (hp->primer) {
    if ((rc = step(0, 1)) != GB_OK) return rc;
    lstm_epoch_kernel<<<jb, 128, 0, st>>>(jobs, n_jobs, a.loss_sum, a.hit_sum, out_loss, out_acc, -1, hp->epochs);
  }
  for (int e = 0; e < hp->epochs; ++e) {
    for (int w = 0; w < max_windows; w += hp->batch_size)
      if ((rc = step(w, hp->batch_size)) != GB_OK) return rc;
    if (stop != nullptr) run.end_epoch(e, a.loss_sum, a.hit_sum, out_loss, out_acc, st);
    else lstm_epoch_kernel<<<jb, 128, 0, st>>>(jobs, n_jobs, a.loss_sum, a.hit_sum, out_loss, out_acc, e, hp->epochs);
  }
  if (stop != nullptr) run.finish(st);
  cudaGraphExecDestroy(gexec);  // the enqueued replays keep what they need
  GB_CUDA_CHECK(cudaGetLastError());
  return GB_OK;
}

int gb_lstm_fit_opt(const gb_lstmnet* net, float* params, float* adam_m, float* adam_v, int32_t* adam_t, const gb_job* jobs,
                    int32_t n_jobs, int32_t max_windows, const float* x, const float* y, const gb_lstm_fit_hparams* hp, void* workspace,
                    float* out_loss, float* out_acc, int32_t loss, const gb_optimizer* opt, void* stream) {
  return launch_fit(net, params, adam_m, adam_v, adam_t, jobs, n_jobs, max_windows, x, y, hp, workspace, out_loss, out_acc, loss, opt,
                    nullptr, nullptr, nullptr, nullptr, stream);
}

int gb_lstm_fit_stop(const gb_lstmnet* net, float* params, float* adam_m, float* adam_v, int32_t* adam_t, const gb_job* jobs,
                     int32_t n_jobs, int32_t max_windows, const float* x, const float* y, const gb_lstm_fit_hparams* hp, void* workspace,
                     float* out_loss, float* out_acc, int32_t loss, const gb_optimizer* opt, const gb_fit_stop* stop, float* best_params,
                     int32_t* out_epochs, int32_t* out_best_epoch, void* stream) {
  return launch_fit(net, params, adam_m, adam_v, adam_t, jobs, n_jobs, max_windows, x, y, hp, workspace, out_loss, out_acc, loss, opt,
                    stop, best_params, out_epochs, out_best_epoch, stream);
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
