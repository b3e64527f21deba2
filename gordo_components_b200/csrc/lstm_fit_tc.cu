// K3-fit on the Hopper tensor cores: the training of lstm_fit.cu (same primer step, epochs, batches in window order, losses,
// accuracy, Adam and launch sequence) for batches of up to MAX_BATCH windows.  lstm_fit.cu keeps batches of <= 32 on fp32 CUDA
// cores; this family tiles the batch in TM = 64-window tiles and runs the three contractions of a step on wgmma:
//   forward   z_t = [x_t | h_{t-1} | 1] [K; U; b]                 grid (ceil(u/16), batch tiles, jobs): 16 units x 4 gates per tile
//   backward  [dx_t | dh_{t-1}] = dz_t [K; U]^T                   grid (ceil(cols/64), batch tiles, jobs)
//   weights   d[K; U; b] = sum_{t,b} [x_t | h_{t-1} | 1]^T dz_t   grid (ceil(4u/64), ceil((in+u+1)/64), jobs), reduction length L * batch
// (the bias rides as a row of ones in the A operand, so the parameter block [K; U; b] is one matrix of in + u + 1 rows).
//
// All three are the same tile routine (mma_step): a 64 x 64 fp32 accumulator in registers, fed TK = 32 reduction rows at a time.
// The operands are read through accessors with whatever strides the GEMM needs and written by ordinary stores into shared
// memory, A row-major and B as the K-major image wgmma takes for TF32, so no operand is ever transposed in global memory.
//
// Precision: the gradients are unbounded, so the FP16-pair scheme of the inference kernels does not apply.  Each operand is
// split v = hi + lo with hi = v rounded to TF32 (10-bit mantissa) and lo = v - hi (exact in fp32, read by the tensor core as TF32),
// and D += hi*hi + hi*lo + lo*hi: three m64n64k8 MMAs per 8 reduction rows, fp32 accumulation.  The dropped lo*lo term and the
// truncation of lo are ~2^-21 relative per product, the order of fp32 rounding.  The cell update, gate gradients and the Dense
// head (loss, loss gradient, accuracy) stay in fp32 with expf / tanhf as in lstm_fit.cu.
//
// The head runs as two launches so that any batch fits: per 16-row slice of a batch, the Dense layer, loss, its gradient
// (kept in the workspace), accuracy and dh of the top layer; then per job the Dense gradients, reduced over the whole batch in
// row order, and the slice sums added in slice order.  No atomics: every launch is deterministic.
#include "gb_common.cuh"
#include "gb_sm90.cuh"
#include "lstm_fit_stop.cuh"

namespace {

using namespace gb::sm90;

constexpr int TM = 64;           // batch rows per tile (wgmma M)
constexpr int TN = 64;           // output columns per tile (wgmma N)
constexpr int TK = 32;           // reduction rows staged per mma_step
constexpr int MAX_BATCH = 256;   // largest batch_size accepted
constexpr int HEAD_ROWS = 16;    // batch rows per CTA of the head
constexpr int LSTM_MAX_UNITS = 512;
constexpr int LSTM_MAX_FEATURES = 512;

struct Lay {
  int in, u;       // input width, units
  int act;
  long kofs;       // offset of [K; U] (rows in + u, 4u columns) in the parameter vector; bias follows
  long zofs, cofs, hofs, dhofs, nxofs;  // workspace offsets (floats, per job): gates [L][Bp][4u], c / h [L][Bp][u], dh_seq [L][Bp][u], (dh_next, dc_next) [2][Bp][u]
};

struct FitArgs {
  int n_layers, L, F, T_out, out_act, lookahead;
  int Bp;           // batch rows the workspace holds per timestep: batch_size rounded up to TM
  Lay lay[GB_MAX_LAYERS];
  long dofs;        // Dense kernel offset in the parameter vector
  long pstride, ws_stride;  // floats per slot / per job
  long gofs;        // gradient vector offset in the job workspace
  long topdh;       // [Bp][u_top] dh of the last LSTM layer at t = L-1
  long doutofs;     // [Bp][T_out] d(loss)/d(Dense pre-activation)
  long partofs;     // [Bp / HEAD_ROWS][2] loss and hit sums per head slice
  float* params;
  float *adam_m, *adam_v;
  int* adam_t;
  const gb_job* jobs;
  const float *x, *y;
  float* ws;
  float *loss_sum, *hit_sum;  // [n_jobs]
  const int* step;            // device: {first window, batch size} of the optimizer step being replayed
  float lr, b1, b2, eps;
  int loss;
  gb_optimizer opt;  // another optimizer than plain Adam (tc_opt_kernel)
};

__device__ __forceinline__ float sigm(float z) { return 1.f / (1.f + expf(-z)); }
__device__ __forceinline__ int job_batch(const gb_job& job, int win0, int bsz) { return max(0, min(bsz, job.n_rows - win0)); }

__device__ __forceinline__ float tf32_hi(float v) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(v));
  return __uint_as_float(r);
}

// ---------------------------------------------------------------------------------------------- the tile routine
struct __align__(128) Tile {
  float bhi[TK / 4][TN][4];  // B as wgmma's K-major TF32 image: core matrices of 8 n x 4 k (128 B), 8-n groups 128 B apart,
  float blo[TK / 4][TN][4];  // 4-k groups TN * 16 B apart
  float a[TM][TK + 4];       // A row-major; the pad makes the fragment reads conflict-free
};

__device__ __forceinline__ void fence_acc(float (&d)[32]) {
#pragma unroll
  for (int i = 0; i < 32; ++i) fence_reg(d[i]);
}

// D[64][64] += A[64][TK] B[TK][64] for the CTA's one warpgroup.  fa(m, k) and fb(k, n) return the operands, 0 outside the
// matrices.  A_M_FAST / B_K_FAST say which index runs across consecutive threads while staging (the one contiguous in memory).
// Thread (warp w, lane 4 g + t) holds d[4 j + 2 h + e] = D[16 w + g + 8 h][8 j + 2 t + e].
template <bool A_M_FAST, bool B_K_FAST, class FA, class FB>
__device__ __forceinline__ void mma_step(Tile& s, const FA& fa, const FB& fb, float (&d)[32]) {
  const int tid = threadIdx.x;
#pragma unroll 4
  for (int i = tid; i < TM * TK; i += 128) {
    const int m = A_M_FAST ? (i & (TM - 1)) : (i / TK), k = A_M_FAST ? (i / TM) : (i & (TK - 1));
    s.a[m][k] = fa(m, k);
  }
#pragma unroll 4
  for (int i = tid; i < TK * TN; i += 128) {
    const int k = B_K_FAST ? (i & (TK - 1)) : (i / TN), n = B_K_FAST ? (i / TK) : (i & (TN - 1));
    const float v = fb(k, n), hi = tf32_hi(v);
    s.bhi[k >> 2][n][k & 3] = hi;
    s.blo[k >> 2][n][k & 3] = v - hi;
  }
  fence_proxy_async();  // the generic-proxy stores above are read by the tensor cores
  __syncthreads();
  const int lane = tid & 31, g = lane >> 2, t = lane & 3, r = 16 * (tid >> 5) + g;
  uint32_t ahi[TK / 8][4], alo[TK / 8][4];  // TF32 A fragment: (row g, col t), (g + 8, t), (g, t + 4), (g + 8, t + 4)
#pragma unroll
  for (int ks = 0; ks < TK / 8; ++ks) {
    const float v[4] = {s.a[r][8 * ks + t], s.a[r + 8][8 * ks + t], s.a[r][8 * ks + t + 4], s.a[r + 8][8 * ks + t + 4]};
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float hi = tf32_hi(v[q]);
      ahi[ks][q] = __float_as_uint(hi);
      alo[ks][q] = __float_as_uint(v[q] - hi);
    }
  }
  const uint32_t bh = smem_u32(s.bhi), bl = smem_u32(s.blo);
  constexpr uint32_t LBO = TN * 16, STEP = 2 * TN * 16;
  wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < TK / 8; ++ks) {  // the small terms first
    wgmma_rs_tf32_n64(d, alo[ks], desc_noswizzle(bh + ks * STEP, LBO, 128), 1);
    wgmma_rs_tf32_n64(d, ahi[ks], desc_noswizzle(bl + ks * STEP, LBO, 128), 1);
    wgmma_rs_tf32_n64(d, ahi[ks], desc_noswizzle(bh + ks * STEP, LBO, 128), 1);
  }
  wgmma_commit();
  wgmma_wait<0>();
  fence_acc(d);
  __syncthreads();  // the tile buffers are refilled by the next step
}

// ---------------------------------------------------------------------------------------------- forward cell
// grid (ceil(u/16), Bp/64, n_jobs), 128 threads.  Tile column 16 q + j is gate q (i, f, c, o) of unit u0 + j, so every thread
// holds all four gates of its units: the cell update runs on the accumulator.
__global__ void __launch_bounds__(128) tc_fwd_kernel(const FitArgs a, int l, int t) {
  const gb_job job = a.jobs[blockIdx.z];
  const int nb = job_batch(job, a.step[0], a.step[1]);
  const int b0 = blockIdx.y * TM;
  if (b0 >= nb) return;
  const Lay ly = a.lay[l];
  const int u = ly.u, in = ly.in, KK = in + u, u4 = 4 * u, Bp = a.Bp;
  const int u0 = blockIdx.x * 16;
  float* ws = a.ws + (long)blockIdx.z * a.ws_stride;
  const float* P = a.params + (long)job.slot * a.pstride + ly.kofs;  // [K; U] rows, then the bias row
  const float* hprev = ws + ly.hofs + (long)(t - 1) * Bp * u;
  const float* below = l > 0 ? ws + a.lay[l - 1].hofs + (long)t * Bp * in : nullptr;
  const float* xt = a.x + (job.x_row + a.step[0] + t) * (long)a.F;  // window b's row at time t: xt + b * F
  __shared__ Tile s;
  float d[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) d[i] = 0.f;
  for (int k0 = 0; k0 <= KK; k0 += TK) {
    const auto fa = [&](int m, int kk) -> float {
      const int b = b0 + m, k = k0 + kk;
      if (b >= nb || k > KK) return 0.f;
      if (k == KK) return 1.f;
      if (k < in) return l == 0 ? __ldg(xt + (long)b * a.F + k) : below[(long)b * in + k];
      return t > 0 ? hprev[(long)b * u + (k - in)] : 0.f;
    };
    const auto fb = [&](int kk, int n) -> float {
      const int k = k0 + kk, un = u0 + (n & 15);
      return (k <= KK && un < u) ? __ldg(P + (long)k * u4 + (n >> 4) * u + un) : 0.f;
    };
    mma_step<false, false>(s, fa, fb, d);
  }
  float* Z = ws + ly.zofs + (long)t * Bp * u4;
  float* C = ws + ly.cofs + (long)t * Bp * u;
  float* H = ws + ly.hofs + (long)t * Bp * u;
  const float* Cp = ws + ly.cofs + (long)(t - 1) * Bp * u;
  const int lane = threadIdx.x & 31, r = 16 * (threadIdx.x >> 5) + (lane >> 2), tq = lane & 3;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int b = b0 + r + 8 * h;
    if (b >= nb) continue;
#pragma unroll
    for (int jj = 0; jj < 2; ++jj)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int un = u0 + 8 * jj + 2 * tq + e;
        if (un >= u) continue;
        const int o = 4 * jj + 2 * h + e;  // gate q sits at d[8 q + o]
        const float ig = sigm(d[o]), fg = sigm(d[8 + o]), gg = gb::apply_act(ly.act, d[16 + o]), og = sigm(d[24 + o]);
        const float cp = t > 0 ? Cp[(long)b * u + un] : 0.f;
        const float c = fmaf(fg, cp, ig * gg);
        float* zr = Z + (long)b * u4;
        zr[un] = ig; zr[u + un] = fg; zr[2 * u + un] = gg; zr[3 * u + un] = og;
        C[(long)b * u + un] = c;
        H[(long)b * u + un] = og * gb::apply_act(ly.act, c);
      }
  }
}

// ---------------------------------------------------------------------------------------------- Dense head, loss, its gradients
// grid (Bp / HEAD_ROWS, n_jobs), 256 threads: one 16-row slice of the batch.  Dynamic smem: h [16][u], dout [16][T], yhat [16][T].
__global__ void __launch_bounds__(256) tc_head_rows_kernel(const FitArgs a) {
  const gb_job job = a.jobs[blockIdx.y];
  const int nb = job_batch(job, a.step[0], a.step[1]);
  const int b0 = blockIdx.x * HEAD_ROWS;
  if (b0 >= nb) return;
  const int nr = min(HEAD_ROWS, nb - b0);
  extern __shared__ float sm[];
  const Lay top = a.lay[a.n_layers - 1];
  const int u = top.u, T = a.T_out;
  float* sh = sm;
  float* sd = sh + HEAD_ROWS * u;
  float* sy = sd + HEAD_ROWS * T;
  __shared__ float red[256];
  __shared__ float shit[HEAD_ROWS];
  float* ws = a.ws + (long)blockIdx.y * a.ws_stride;
  const float* P = a.params + (long)job.slot * a.pstride + a.dofs;  // Wd [u][T], bd [T]
  const float* H = ws + top.hofs + ((long)(a.L - 1) * a.Bp + b0) * u;
  float* Dout = ws + a.doutofs + (long)b0 * T;
  const int tid = threadIdx.x;
  for (int i = tid; i < nr * u; i += 256) sh[i] = H[i];
  __syncthreads();
  const float inv = 2.0f / (float)(nb * T);
  const float linv = 1.0f / (float)(nb * T);
  const long yrow0 = job.x_row + a.step[0] + b0 + a.L - 1 + a.lookahead;
  float lsum = 0.f;
  for (int i = tid; i < nr * T; i += 256) {
    const int b = i / T, o = i - b * T;
    float z = __ldg(P + (long)u * T + o);
    for (int k = 0; k < u; ++k) z = fmaf(sh[b * u + k], __ldg(P + (long)k * T + o), z);
    const float yh = gb::apply_act(a.out_act, z);
    const float tgt = __ldg(a.y + (yrow0 + b) * T + o);
    sy[i] = yh;
    float g;
    if (a.loss == GB_LOSS_MSE) {
      const float dd = yh - tgt;
      lsum += dd * dd;
      g = inv * dd * gb::act_grad_from_output(a.out_act, yh);
    } else {
      lsum += gb::loss_value(a.loss, yh, tgt);
      g = linv * gb::loss_grad(a.loss, yh, tgt) * gb::act_grad_from_output(a.out_act, yh);
    }
    sd[i] = g;
    Dout[i] = g;
  }
  red[tid] = lsum;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (tid < s) red[tid] += red[tid + s];
    __syncthreads();
  }
  // accuracy (metrics=["accuracy"] on 2-D float targets: argmax match; width 1: thresholded match)
  if (tid < nr) {
    const float* tg = a.y + (yrow0 + tid) * T;
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
    shit[tid] = hit;
  }
  __syncthreads();
  if (tid == 0) {
    float hits = 0.f;
    for (int b = 0; b < nr; ++b) hits += shit[b];
    ws[a.partofs + 2 * blockIdx.x] = red[0];
    ws[a.partofs + 2 * blockIdx.x + 1] = hits;
  }
  // dh of the last LSTM layer at t = L-1: dh[b][k] = sum_o dout[b][o] Wd[k][o]
  float* DH = ws + a.topdh + (long)b0 * u;
  for (int i = tid; i < nr * u; i += 256) {
    const int b = i / u, k = i - b * u;
    float g = 0.f;
    for (int o = 0; o < T; ++o) g = fmaf(sd[b * T + o], __ldg(P + (long)k * T + o), g);
    DH[i] = g;
  }
}

// grid (ceil((u + 1) T / 256), n_jobs), 256 threads: dWd[k][o] = sum_b h[b][k] dout[b][o], dbd[o] = sum_b dout[b][o] over the
// whole batch in row order; block 0 adds the slices' loss and hit sums to the epoch totals.
__global__ void __launch_bounds__(256) tc_head_grad_kernel(const FitArgs a) {
  const gb_job job = a.jobs[blockIdx.y];
  const int nb = job_batch(job, a.step[0], a.step[1]);
  if (nb == 0) return;
  const Lay top = a.lay[a.n_layers - 1];
  const int u = top.u, T = a.T_out;
  float* ws = a.ws + (long)blockIdx.y * a.ws_stride;
  const float* H = ws + top.hofs + (long)(a.L - 1) * a.Bp * u;
  const float* Dout = ws + a.doutofs;
  float* G = ws + a.gofs + a.dofs;
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i < u * T) {
    const int k = i / T, o = i - k * T;
    float g = 0.f;
    for (int b = 0; b < nb; ++b) g = fmaf(H[(long)b * u + k], Dout[(long)b * T + o], g);
    G[i] = g;
  } else if (i < (u + 1) * T) {
    const int o = i - u * T;
    float g = 0.f;
    for (int b = 0; b < nb; ++b) g += Dout[(long)b * T + o];
    G[i] = g;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    float ls = 0.f, hs = 0.f;
    for (int s = 0; s * HEAD_ROWS < nb; ++s) {
      ls += ws[a.partofs + 2 * s];
      hs += ws[a.partofs + 2 * s + 1];
    }
    a.loss_sum[blockIdx.y] += ls / (float)(nb * T) * (float)nb;
    a.hit_sum[blockIdx.y] += hs;
  }
}

// ---------------------------------------------------------------------------------------------- backward: gate gradients
// grid (ceil(Bp*u/256), n_jobs).  Overwrites the saved gates of (l, t) with dz, updates dc_next.
__global__ void __launch_bounds__(256) tc_bwd_gates_kernel(const FitArgs a, int l, int t) {
  const gb_job job = a.jobs[blockIdx.y];
  const int nb = job_batch(job, a.step[0], a.step[1]);
  if (nb == 0) return;
  const Lay ly = a.lay[l];
  const int u = ly.u, u4 = 4 * u, Bp = a.Bp;
  const int i = blockIdx.x * 256 + threadIdx.x;
  const int b = i / u, un = i - b * u;
  if (b >= nb) return;
  float* ws = a.ws + (long)blockIdx.y * a.ws_stride;
  float* Z = ws + ly.zofs + (long)t * Bp * u4 + (long)b * u4;
  const float ig = Z[un], fg = Z[u + un], gg = Z[2 * u + un], og = Z[3 * u + un];
  const long bu = (long)b * u + un;
  const float c = ws[ly.cofs + (long)t * Bp * u + bu];
  const float cp = t > 0 ? ws[ly.cofs + (long)(t - 1) * Bp * u + bu] : 0.f;
  float* nx = ws + ly.nxofs;  // dh_next [Bp][u], dc_next [Bp][u]
  const bool last_t = t == a.L - 1;
  float dh = last_t ? 0.f : nx[bu];
  if (l == a.n_layers - 1) {
    if (last_t) dh += ws[a.topdh + bu];
  } else {
    dh += ws[ly.dhofs + (long)t * Bp * u + bu];
  }
  const float ac = gb::apply_act(ly.act, c);
  const float dc = dh * og * gb::act_grad_from_output(ly.act, ac) + (last_t ? 0.f : nx[(long)Bp * u + bu]);
  Z[un] = dc * gg * ig * (1.f - ig);
  Z[u + un] = dc * cp * fg * (1.f - fg);
  Z[2 * u + un] = dc * ig * gb::act_grad_from_output(ly.act, gg);
  Z[3 * u + un] = dh * ac * og * (1.f - og);
  nx[(long)Bp * u + bu] = dc * fg;
}

// ---------------------------------------------------------------------------------------------- backward: [dx_t | dh_{t-1}] = dz_t [K; U]^T
// grid (ceil(cols/64), Bp/64, n_jobs) over the columns that are needed (layer 0 has no dx), 128 threads.
__global__ void __launch_bounds__(128) tc_bwd_input_kernel(const FitArgs a, int l, int t) {
  const gb_job job = a.jobs[blockIdx.z];
  const int nb = job_batch(job, a.step[0], a.step[1]);
  const int b0 = blockIdx.y * TM;
  if (b0 >= nb) return;
  const Lay ly = a.lay[l];
  const int u = ly.u, in = ly.in, KK = in + u, u4 = 4 * u, Bp = a.Bp;
  const int kbase = (l == 0 ? in : 0) + blockIdx.x * TN;  // first output column (row of [K; U]) of this CTA
  float* ws = a.ws + (long)blockIdx.z * a.ws_stride;
  const float* P = a.params + (long)job.slot * a.pstride + ly.kofs;
  const float* Z = ws + ly.zofs + (long)t * Bp * u4;
  __shared__ Tile s;
  float d[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) d[i] = 0.f;
  for (int c0 = 0; c0 < u4; c0 += TK) {
    const auto fa = [&](int m, int cc) -> float {
      const int b = b0 + m, c = c0 + cc;
      return (b < nb && c < u4) ? Z[(long)b * u4 + c] : 0.f;
    };
    const auto fb = [&](int cc, int n) -> float {
      const int c = c0 + cc, k = kbase + n;
      return (k < KK && c < u4) ? __ldg(P + (long)k * u4 + c) : 0.f;
    };
    mma_step<false, true>(s, fa, fb, d);
  }
  const int lane = threadIdx.x & 31, r = 16 * (threadIdx.x >> 5) + (lane >> 2), tq = lane & 3;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int b = b0 + r + 8 * h;
    if (b >= nb) continue;
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int k = kbase + 8 * j + 2 * tq + e;
        if (k >= KK) continue;
        const float v = d[4 * j + 2 * h + e];
        if (k < in) ws[a.lay[l - 1].dhofs + (long)t * Bp * in + (long)b * in + k] = v;  // the layer below's dh at time t
        else ws[ly.nxofs + (long)b * u + (k - in)] = v;                                    // dh_next of this layer
      }
  }
}

// ---------------------------------------------------------------------------------------------- weight gradients
// d[K; U; b][k][c] = sum_{t,b} [x_t | h_{t-1} | 1][b][k] dz_t[b][c]: grid (ceil(4u/64), ceil((in+u+1)/64), n_jobs), 128 threads,
// a 64 x 64 tile of rows k x columns c with the reduction over (t, b) in steps of TK windows.
__global__ void __launch_bounds__(128) tc_wgrad_kernel(const FitArgs a, int l) {
  const gb_job job = a.jobs[blockIdx.z];
  const int nb = job_batch(job, a.step[0], a.step[1]);
  if (nb == 0) return;
  const Lay ly = a.lay[l];
  const int u = ly.u, in = ly.in, KK = in + u, u4 = 4 * u, Bp = a.Bp;
  const int c0 = blockIdx.x * TN, k0 = blockIdx.y * TM;
  float* ws = a.ws + (long)blockIdx.z * a.ws_stride;
  float* G = ws + a.gofs + ly.kofs;
  __shared__ Tile s;
  float d[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) d[i] = 0.f;
  for (int t = 0; t < a.L; ++t) {
    const float* Z = ws + ly.zofs + (long)t * Bp * u4;
    const float* below = l > 0 ? ws + a.lay[l - 1].hofs + (long)t * Bp * in : nullptr;
    const float* hprev = ws + ly.hofs + (long)(t - 1) * Bp * u;
    const float* xt = a.x + (job.x_row + a.step[0] + t) * (long)a.F;
    for (int r0 = 0; r0 < nb; r0 += TK) {
      const auto fa = [&](int m, int rr) -> float {
        const int k = k0 + m, b = r0 + rr;
        if (b >= nb || k > KK) return 0.f;
        if (k == KK) return 1.f;
        if (k < in) return l == 0 ? __ldg(xt + (long)b * a.F + k) : below[(long)b * in + k];
        return t > 0 ? hprev[(long)b * u + (k - in)] : 0.f;
      };
      const auto fb = [&](int rr, int n) -> float {
        const int b = r0 + rr, c = c0 + n;
        return (b < nb && c < u4) ? Z[(long)b * u4 + c] : 0.f;
      };
      mma_step<true, false>(s, fa, fb, d);
    }
  }
  const int lane = threadIdx.x & 31, r = 16 * (threadIdx.x >> 5) + (lane >> 2), tq = lane & 3;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int k = k0 + r + 8 * h;
    if (k > KK) continue;
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int c = c0 + 8 * j + 2 * tq + e;
        if (c < u4) G[(long)k * u4 + c] = d[4 * j + 2 * h + e];
      }
  }
}

// ---------------------------------------------------------------------------------------------- Adam and step bookkeeping (as lstm_fit.cu)
__global__ void __launch_bounds__(256) tc_adam_kernel(const FitArgs a, long n_params) {
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
// Every other optimizer than plain Adam (gb::opt_update; state slots 0 / 1 = adam_m / adam_v), captured in place of tc_adam_kernel.
// The per-step scalars come from the slot's step count, once per CTA (for Nadam a product over the slot's steps, a few cycles each).
__global__ void __launch_bounds__(256) tc_opt_kernel(const FitArgs a, long n_params) {
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
__global__ void tc_bump_kernel(const FitArgs a, int n_jobs) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n_jobs && job_batch(a.jobs[j], a.step[0], a.step[1]) > 0) a.adam_t[a.jobs[j].slot] += 1;
}
__global__ void tc_set_step_kernel(int* step, int win0, int bsz) {
  step[0] = win0;
  step[1] = bsz;
}
__global__ void tc_epoch_kernel(const gb_job* jobs, int n_jobs, float* loss_sum, float* hit_sum, float* out_loss, float* out_acc, int epoch, int epochs) {
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

int padded_batch(int batch_size) { return (batch_size + TM - 1) / TM * TM; }

// workspace layout of one job (floats) for batches of up to Bp windows; returns the total
long layout(const gb_lstmnet* net, int Bp, FitArgs* a) {
  long ofs = 0, pofs = 0;
  int in = net->n_features;
  const long L = net->lookback;
  a->Bp = Bp;
  for (int l = 0; l < net->n_layers; ++l) {
    const int u = net->units[l];
    Lay& ly = a->lay[l];
    ly.in = in; ly.u = u; ly.act = net->act[l];
    ly.kofs = pofs;
    pofs += 4L * u * (in + u + 1);
    ly.zofs = ofs; ofs += L * Bp * 4 * u;
    ly.cofs = ofs; ofs += L * Bp * u;
    ly.hofs = ofs; ofs += L * Bp * u;
    ly.dhofs = ofs; ofs += (l + 1 < net->n_layers) ? L * Bp * u : 0;
    ly.nxofs = ofs; ofs += 2L * Bp * u;
    in = u;
  }
  a->dofs = pofs;
  a->topdh = ofs; ofs += (long)Bp * in;
  a->doutofs = ofs; ofs += (long)Bp * net->n_features_out;
  a->partofs = ofs; ofs += 2L * (Bp / HEAD_ROWS);
  a->gofs = ofs; ofs += (long)gb_lstm_param_stride(net);
  return (ofs + 3) / 4 * 4;
}

}  // namespace

extern "C" {

size_t gb_lstm_fit_tc_workspace_bytes(const gb_lstmnet* net, int32_t n_jobs, int32_t batch_size) {
  if (validate(net) != GB_OK || n_jobs < 0 || batch_size < 1 || batch_size > MAX_BATCH) return 0;
  FitArgs a{};
  return (size_t)(layout(net, padded_batch(batch_size), &a) * (long)n_jobs + 2L * n_jobs + 4) * sizeof(float);
}

int gb_lstm_fit_tc(const gb_lstmnet* net, float* params, float* adam_m, float* adam_v, int32_t* adam_t, const gb_job* jobs,
                   int32_t n_jobs, int32_t max_windows, const float* x, const float* y, const gb_lstm_fit_hparams* hp, void* workspace,
                   float* out_loss, float* out_acc, int32_t loss, void* stream) {
  return gb_lstm_fit_tc_opt(net, params, adam_m, adam_v, adam_t, jobs, n_jobs, max_windows, x, y, hp, workspace, out_loss, out_acc, loss,
                            nullptr, stream);
}

// gb_lstm_fit_tc_opt (stop NULL: the step graph and launches as they have always been) and gb_lstm_fit_tc_stop
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
  GB_REQUIRE(hp->batch_size <= MAX_BATCH, GB_E_SHAPE, "batch_size=%d: the tensor-core LSTM fit handles batches of at most %d windows",
             hp->batch_size, MAX_BATCH);
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
  a.ws_stride = layout(net, padded_batch(hp->batch_size), &a);
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
  const int u_top = net->units[net->n_layers - 1], T = net->n_features_out;
  const size_t head_smem = (size_t)(HEAD_ROWS * u_top + 2 * HEAD_ROWS * T) * sizeof(float);
  GB_CUDA_CHECK(cudaFuncSetAttribute(tc_head_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)head_smem));
  const int jb = (n_jobs + 127) / 128;
  const int nbt = a.Bp / TM;

  int* d_step = reinterpret_cast<int*>(a.hit_sum + n_jobs);
  a.step = d_step;
  const lstm_stop::Run run(workspace, gb_lstm_fit_tc_workspace_bytes(net, n_jobs, hp->batch_size), jobs, n_jobs, hp->epochs, out_epochs,
                           out_best_epoch, params, best_params, a.pstride, n_params);
  if (stop != nullptr) {
    run.init(stop, st);
    a.jobs = run.job_copy;  // a job that stops gets n_rows 0 here, so job_batch gives it no windows
  }
  // the launch sequence of one optimizer step, captured once and replayed per step as in gb_lstm_fit_loss
  cudaGraphExec_t gexec = nullptr;
  rc = capture_step(&gexec, stop != nullptr ? run.live : nullptr, [&](cudaStream_t st) {
    for (int t = 0; t < a.L; ++t)
      for (int l = 0; l < a.n_layers; ++l) tc_fwd_kernel<<<dim3((a.lay[l].u + 15) / 16, nbt, n_jobs), 128, 0, st>>>(a, l, t);
    tc_head_rows_kernel<<<dim3(a.Bp / HEAD_ROWS, n_jobs), 256, head_smem, st>>>(a);
    tc_head_grad_kernel<<<dim3(((u_top + 1) * T + 255) / 256, n_jobs), 256, 0, st>>>(a);
    for (int t = a.L - 1; t >= 0; --t)
      for (int l = a.n_layers - 1; l >= 0; --l) {
        const Lay& ly = a.lay[l];
        tc_bwd_gates_kernel<<<dim3((a.Bp * ly.u + 255) / 256, n_jobs), 256, 0, st>>>(a, l, t);
        const int cols = l == 0 ? ly.u : ly.in + ly.u;
        if (t > 0 || l > 0) tc_bwd_input_kernel<<<dim3((cols + TN - 1) / TN, nbt, n_jobs), 128, 0, st>>>(a, l, t);
      }
    for (int l = 0; l < a.n_layers; ++l) {
      const Lay& ly = a.lay[l];
      tc_wgrad_kernel<<<dim3((4 * ly.u + TN - 1) / TN, (ly.in + ly.u + 1 + TM - 1) / TM, n_jobs), 128, 0, st>>>(a, l);
    }
    if (use_opt)
      tc_opt_kernel<<<dim3((unsigned)((n_params + 256 * 8 - 1) / (256 * 8)), n_jobs), 256, 0, st>>>(a, n_params);
    else
      tc_adam_kernel<<<dim3((unsigned)((n_params + 256 * 8 - 1) / (256 * 8)), n_jobs), 256, 0, st>>>(a, n_params);
    tc_bump_kernel<<<jb, 128, 0, st>>>(a, n_jobs);
  });
  if (rc != GB_OK) return rc;
  auto step = [&](int win0, int bsz) -> int {
    tc_set_step_kernel<<<1, 1, 0, st>>>(d_step, win0, bsz);
    const cudaError_t ce = cudaGraphLaunch(gexec, st);
    if (ce != cudaSuccess) {
      cudaGraphExecDestroy(gexec);
      gb::set_error("cudaGraphLaunch failed: %s", cudaGetErrorString(ce));
      return GB_E_CUDA;
    }
    return GB_OK;
  };

  tc_epoch_kernel<<<jb, 128, 0, st>>>(jobs, n_jobs, a.loss_sum, a.hit_sum, out_loss, out_acc, -1, hp->epochs);
  if (hp->primer) {
    if ((rc = step(0, 1)) != GB_OK) return rc;
    tc_epoch_kernel<<<jb, 128, 0, st>>>(jobs, n_jobs, a.loss_sum, a.hit_sum, out_loss, out_acc, -1, hp->epochs);
  }
  for (int e = 0; e < hp->epochs; ++e) {
    for (int w = 0; w < max_windows; w += hp->batch_size)
      if ((rc = step(w, hp->batch_size)) != GB_OK) return rc;
    if (stop != nullptr) run.end_epoch(e, a.loss_sum, a.hit_sum, out_loss, out_acc, st);
    else tc_epoch_kernel<<<jb, 128, 0, st>>>(jobs, n_jobs, a.loss_sum, a.hit_sum, out_loss, out_acc, e, hp->epochs);
  }
  if (stop != nullptr) run.finish(st);
  cudaGraphExecDestroy(gexec);  // the enqueued replays keep what they need
  GB_CUDA_CHECK(cudaGetLastError());
  return GB_OK;
}

int gb_lstm_fit_tc_opt(const gb_lstmnet* net, float* params, float* adam_m, float* adam_v, int32_t* adam_t, const gb_job* jobs,
                       int32_t n_jobs, int32_t max_windows, const float* x, const float* y, const gb_lstm_fit_hparams* hp, void* workspace,
                       float* out_loss, float* out_acc, int32_t loss, const gb_optimizer* opt, void* stream) {
  return launch_fit(net, params, adam_m, adam_v, adam_t, jobs, n_jobs, max_windows, x, y, hp, workspace, out_loss, out_acc, loss, opt,
                    nullptr, nullptr, nullptr, nullptr, stream);
}

int gb_lstm_fit_tc_stop(const gb_lstmnet* net, float* params, float* adam_m, float* adam_v, int32_t* adam_t, const gb_job* jobs,
                        int32_t n_jobs, int32_t max_windows, const float* x, const float* y, const gb_lstm_fit_hparams* hp, void* workspace,
                        float* out_loss, float* out_acc, int32_t loss, const gb_optimizer* opt, const gb_fit_stop* stop, float* best_params,
                        int32_t* out_epochs, int32_t* out_best_epoch, void* stream) {
  return launch_fit(net, params, adam_m, adam_v, adam_t, jobs, n_jobs, max_windows, x, y, hp, workspace, out_loss, out_acc, loss, opt,
                    stop, best_params, out_epochs, out_best_epoch, stream);
}

}  // extern "C"
