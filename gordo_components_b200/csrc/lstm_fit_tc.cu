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
#include "lstm_fit_common.cuh"

namespace {

using namespace gb::sm90;

constexpr int TM = 64;           // batch rows per tile (wgmma M)
constexpr int TN = 64;           // output columns per tile (wgmma N)
constexpr int TK = 32;           // reduction rows staged per mma_step
constexpr int MAX_BATCH = 256;   // largest batch_size accepted
constexpr int HEAD_ROWS = 16;    // batch rows per CTA of the head

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

int padded_batch(int batch_size) { return (batch_size + TM - 1) / TM * TM; }

// fit_driver's policy for this family: the batch in TM-row tiles, the head in HEAD_ROWS-row slices
struct TcFit {
  static constexpr int max_batch = MAX_BATCH;
  static constexpr const char* who = "the tensor-core LSTM fit";
  static constexpr int head_rows = HEAD_ROWS;
  static int rows(int batch_size) { return padded_batch(batch_size); }
  size_t head_smem = 0;

  int prepare(const FitArgs& a) {
    head_smem = (size_t)(HEAD_ROWS * a.lay[a.n_layers - 1].u + 2 * HEAD_ROWS * a.T_out) * sizeof(float);
    GB_CUDA_CHECK(cudaFuncSetAttribute(tc_head_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)head_smem));
    return GB_OK;
  }

  void record(const FitArgs& a, int n_jobs, cudaStream_t st) const {
    const int nbt = a.Bp / TM, u_top = a.lay[a.n_layers - 1].u, T = a.T_out;
    for (int t = 0; t < a.L; ++t)
      for (int l = 0; l < a.n_layers; ++l) tc_fwd_kernel<<<dim3((a.lay[l].u + 15) / 16, nbt, n_jobs), 128, 0, st>>>(a, l, t);
    tc_head_rows_kernel<<<dim3(a.Bp / HEAD_ROWS, n_jobs), 256, head_smem, st>>>(a);
    tc_head_grad_kernel<<<dim3(((u_top + 1) * T + 255) / 256, n_jobs), 256, 0, st>>>(a);
    for (int t = a.L - 1; t >= 0; --t)
      for (int l = a.n_layers - 1; l >= 0; --l) {
        const Lay& ly = a.lay[l];
        lstm_bwd_gates_kernel<<<dim3((a.Bp * ly.u + 255) / 256, n_jobs), 256, 0, st>>>(a, l, t);
        const int cols = l == 0 ? ly.u : ly.in + ly.u;
        if (t > 0 || l > 0) tc_bwd_input_kernel<<<dim3((cols + TN - 1) / TN, nbt, n_jobs), 128, 0, st>>>(a, l, t);
      }
    for (int l = 0; l < a.n_layers; ++l) {
      const Lay& ly = a.lay[l];
      tc_wgrad_kernel<<<dim3((4 * ly.u + TN - 1) / TN, (ly.in + ly.u + 1 + TM - 1) / TM, n_jobs), 128, 0, st>>>(a, l);
    }
  }
};

}  // namespace

extern "C" {

size_t gb_lstm_fit_tc_workspace_bytes(const gb_lstmnet* net, int32_t n_jobs, int32_t batch_size) {
  if (gb::validate_lstmnet(net) != GB_OK || n_jobs < 0 || batch_size < 1 || batch_size > MAX_BATCH) return 0;
  FitArgs a{};
  return workspace_bytes(layout(net, padded_batch(batch_size), HEAD_ROWS, &a), n_jobs);
}

int gb_lstm_fit_tc(const gb_lstmnet* net, float* params, float* adam_m, float* adam_v, int32_t* adam_t, const gb_job* jobs,
                   int32_t n_jobs, int32_t max_windows, const float* x, const float* y, const gb_lstm_fit_hparams* hp, void* workspace,
                   float* out_loss, float* out_acc, int32_t loss, void* stream) {
  return gb_lstm_fit_tc_opt(net, params, adam_m, adam_v, adam_t, jobs, n_jobs, max_windows, x, y, hp, workspace, out_loss, out_acc, loss,
                            nullptr, stream);
}

int gb_lstm_fit_tc_opt(const gb_lstmnet* net, float* params, float* adam_m, float* adam_v, int32_t* adam_t, const gb_job* jobs,
                       int32_t n_jobs, int32_t max_windows, const float* x, const float* y, const gb_lstm_fit_hparams* hp, void* workspace,
                       float* out_loss, float* out_acc, int32_t loss, const gb_optimizer* opt, void* stream) {
  return fit_driver(TcFit{}, net, params, adam_m, adam_v, adam_t, jobs, n_jobs, max_windows, x, y, hp, workspace, out_loss, out_acc,
                    loss, opt, nullptr, nullptr, nullptr, nullptr, stream);
}

int gb_lstm_fit_tc_stop(const gb_lstmnet* net, float* params, float* adam_m, float* adam_v, int32_t* adam_t, const gb_job* jobs,
                        int32_t n_jobs, int32_t max_windows, const float* x, const float* y, const gb_lstm_fit_hparams* hp, void* workspace,
                        float* out_loss, float* out_acc, int32_t loss, const gb_optimizer* opt, const gb_fit_stop* stop, float* best_params,
                        int32_t* out_epochs, int32_t* out_best_epoch, void* stream) {
  return fit_driver(TcFit{}, net, params, adam_m, adam_v, adam_t, jobs, n_jobs, max_windows, x, y, hp, workspace, out_loss, out_acc,
                    loss, opt, stop, best_params, out_epochs, out_best_epoch, stream);
}

}  // extern "C"
