// K3, variant 2: LSTM autoencoder prediction on the Hopper tensor cores (warpgroup MMA, TMA), machine-batched.
//
// Replaces KerasLSTMBaseEstimator.predict (gordo/machine/model/models.py:618-660) for the stacks of
// factories/lstm_autoencoder.py:72-103 (layer widths are padded to multiples of 64 internally; lstm_symmetric's 256/128/64
// defaults -- BASELINE configs[3] -- need no padding).  Windows are index arithmetic, never materialised (:713-793).
//
// 335 MFLOP per 144 x 128 window is tensor-core work.  One launch advances EVERY window of EVERY job by one (layer,
// timestep): a CTA owns a tile of 128 windows x 64 units and computes the four gate pre-activations
//      z[128, 4 x 64] = [h_below,t | h_own,t-1] (128 x K)  .  [K; U]^T (K x 256)
// as wgmma (m64n256k16, two consumer warpgroups of 64 windows each) with both operands brought to shared memory by TMA
// (SWIZZLE_128B K-major boxes, a ring of STAGES chunks of K = 64 fed by a producer warp), accumulates in registers, and
// finishes the cell in the epilogue: gates, c_t, h_t, with h_t written straight back as the next launches' A operand.  The
// recurrent state of all windows lives in HBM (h as an FP16 pair, c in fp32): per timestep that is a few GB of traffic
// against tens of TFLOP of contraction.
//
// Numerics (1e-4 parity): h in (-1, 1) and the weights are split into FP16 pairs (a = a1 + a2, 22 significant bits) and
// every product is formed as a2*w1 + a1*w2 + a1*w1 with fp32 accumulation -- the scheme of ffae_infer_tc.cu's layers >= 1.
// That bound on h holds for tanh and sigmoid cells only: relu and linear cells have an unbounded h that overflows FP16, so
// gb_lstm_tc_supported refuses them (they run on the fp32 kernel, lstm_infer.cu).
// The raw input x (any magnitude) never enters an FP16 operand: its projection x.K0 + b0 is computed once per x row of each
// job (not per window) in fp32 on the CUDA cores and added in layer 0's epilogue.  Each job keeps its own projection, made with
// its own slot's weights, so jobs of different slots may read the same x rows.
#include <cuda.h>
#include <cuda_fp16.h>
#include "gb_common.cuh"
#include "gb_sm90.cuh"

namespace {

using namespace gb::sm90;

constexpr int TILE = 128;            // windows per CTA
constexpr int UB = 64;               // units per CTA
constexpr int NCOL = 4 * UB;         // gate columns per CTA (wgmma N)
constexpr int KC = 64;               // K elements per pipeline chunk = one 128-byte swizzle row of FP16
constexpr int ROW_BYTES = KC * 2;
constexpr int A_BOX = TILE * ROW_BYTES;  // bytes: 128 rows x KC FP16
constexpr int B_BOX = NCOL * ROW_BYTES;  // bytes: 256 rows x KC FP16
constexpr int STAGE_BYTES = 2 * A_BOX + 2 * B_BOX;  // hi and lo images of both operands: 96 KB
constexpr int STAGES = 2;
constexpr int CONSUMERS = 2;                         // warpgroups: windows 0..63 and 64..127 of the tile
constexpr int NTHREADS = 128 * CONSUMERS + 32;       // + one producer warp

struct TcLayerArgs {
  int u, kc_below, kc_own;           // units; K chunks coming from the layer below / from this layer's own h
  int act;
  int t, n_items;                    // n_items counts (window tile, unit block)
  const int4* tiles;                 // per flat window tile: {slot, windows of the job from this tile on, job, tile within the job}
  const float* bias;                 // [n_slots][4u] reordered (layers >= 1; layer 0's bias lives in xk)
  const float* xk;                   // layer 0: input projection of each job's own x rows, [128-row block][4u reordered][128]
  int xk_pad;                        // job j's xk blocks begin at tile_base[j] + j * xk_pad (its tiles, plus the lookback's rows)
  float* c;                          // [tile][u][128 windows]
  __half *h_out_hi, *h_out_lo;       // [rows][u]
};

// sigmoid through ex2.approx + rcp.approx (~2e-7 absolute error, exact limits); used by the cells whose activation is not tanh
__device__ __forceinline__ float sigm(float z) {
  float e, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-1.4426950408889634f * z));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(e + 1.0f));
  return r;
}
// The tanh cell (every factory default) with the quotients merged: the epilogue is bound by the MUFU pipe, so
//   c' = f*c + i*g = [c*(1+ei)*(1+eg) + (eg-1)*(1+ef)] / [(1+ef)*(1+ei)*(1+eg)],   h = o*tanh(c') = (ec-1) / [(1+eo)*(1+ec)]
// with ei = e^-zi, ef = e^-zf, eo = e^-zo, eg = e^2zg, ec = e^2c' costs five ex2 and two rcp instead of five and five.  The
// exponentials are capped at 2^30 (sigmoid <= 1e-9 / tanh = 1 to fp32 there) so that the products stay finite; min.NaN keeps a NaN a NaN.
__device__ __forceinline__ float ex2_capped(float t) {
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(t));
  asm("min.NaN.ftz.f32 %0, %0, 0f4E800000;" : "+f"(e));  // 2^30
  return e;
}
__device__ __forceinline__ void tanh_cell(float zi, float zf, float zg, float zo, float c_prev, float& c_new, float& h) {
  const float pi = 1.0f + ex2_capped(-1.4426950408889634f * zi), pf = 1.0f + ex2_capped(-1.4426950408889634f * zf);
  const float eg = ex2_capped(2.8853900817779268f * zg), po = 1.0f + ex2_capped(-1.4426950408889634f * zo);
  const float pig = pi * (eg + 1.0f);
  float r1, r2;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r1) : "f"(pig * pf));
  c_new = fmaf(c_prev, pig, (eg - 1.0f) * pf) * r1;
  const float ec = ex2_capped(2.8853900817779268f * c_new);
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r2) : "f"(po * (ec + 1.0f)));
  h = (ec - 1.0f) * r2;
}

// ------------------------------------------------------------------------------------------------ one (layer, timestep) for all windows
// Persistent: gridDim.x CTAs walk the work items (window tile, unit block) in a fixed stride; the producer warp's TMA ring runs
// ahead across items.  An item whose tile holds no window is skipped by every role alike.
// FIRST: layer 0 (the additive term is the per-row input projection, read from global memory); TANH: tanh cell / output activation.
// Both are compile-time so that the epilogue is branch-free.
template <bool FIRST, bool TANH>
__global__ void __launch_bounds__(NTHREADS, 1)
lstm_tc_step_kernel(const __grid_constant__ TcLayerArgs a, const __grid_constant__ CUtensorMap m_below_hi, const __grid_constant__ CUtensorMap m_below_lo,
                    const __grid_constant__ CUtensorMap m_own_hi, const __grid_constant__ CUtensorMap m_own_lo,
                    const __grid_constant__ CUtensorMap m_w_hi, const __grid_constant__ CUtensorMap m_w_lo) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  __shared__ __align__(8) unsigned long long s_bar[2 * STAGES];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));  // SWIZZLE_128B boxes: 1 KB aligned
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const uint32_t sbase = smem_u32(smem);
  const uint32_t bar_full = smem_u32(&s_bar[0]), bar_empty = smem_u32(&s_bar[STAGES]);
  const int u = a.u;
  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(bar_full + 8 * s, 1);
      mbar_init(bar_empty + 8 * s, CONSUMERS);  // one arrival per consumer warpgroup when its MMAs on the stage are complete
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const int n_chunks = a.kc_below + a.kc_own;
  const int nub = u / UB;
  // item -> (tile, ub): the unit blocks of one window tile are neighbours, so CTAs running side by side read the same A operand from L2
  struct Item { int tile, ub, slot, rem, job; bool real; };
  auto item_of = [&](int item) -> Item {
    Item it;
    const int grp = item / nub;
    it.ub = item - grp * nub;
    it.tile = grp;
    const int2 sr = __ldg(reinterpret_cast<const int2*>(a.tiles + grp));  // slot, windows of the job from this tile on
    it.slot = sr.x; it.rem = sr.y;
    it.job = FIRST ? __ldg(reinterpret_cast<const int*>(a.tiles + grp) + 2) : 0;
    it.real = it.rem > 0;
    return it;
  };

  if (warp == CONSUMERS * 4) {
    // ============================== TMA producer (one lane)
    if (lane == 0) {
      int cc = 0;  // chunks issued so far (ring position)
      for (int item = blockIdx.x; item < a.n_items; item += gridDim.x) {
        const Item it = item_of(item);
        if (!it.real) continue;
        const int row0 = it.tile * TILE, wrow0 = it.slot * 4 * u + it.ub * NCOL;
        for (int c = 0; c < n_chunks; ++c, ++cc) {
          const int s = cc % STAGES, round = cc / STAGES;
          if (round > 0) mbar_wait(bar_empty + 8 * s, (round - 1) & 1);
          const uint32_t st = sbase + s * STAGE_BYTES;
          mbar_expect_tx(bar_full + 8 * s, STAGE_BYTES);
          const bool below = c < a.kc_below;
          const int acol = (below ? c : c - a.kc_below) * KC;
          tma_load_2d(st, below ? &m_below_hi : &m_own_hi, acol, row0, bar_full + 8 * s);
          tma_load_2d(st + A_BOX, below ? &m_below_lo : &m_own_lo, acol, row0, bar_full + 8 * s);
          tma_load_2d(st + 2 * A_BOX, &m_w_hi, c * KC, wrow0, bar_full + 8 * s);
          tma_load_2d(st + 2 * A_BOX + B_BOX, &m_w_lo, c * KC, wrow0, bar_full + 8 * s);
        }
      }
    }
  } else {
    // ============================== consumer warpgroup: MMAs of its 64 windows, then gates, cell, h
    // Fragment layout (gb_sm90.cuh): this thread holds windows r0 and r0 + 8 and, for every gate, the unit pairs 8jj + 2t + {0,1}
    // (jj = 0..7) -- accumulator register 4 (8 G + jj) + 2 hr + e is gate G of unit 8jj + 2t + e of window r0 + 8 hr.
    const int wg = warp >> 2, wq = warp & 3, g = lane >> 2, t = lane & 3;
    const int r0 = wg * 64 + wq * 16 + g;  // window row in the tile
    int cc = 0;
    for (int item = blockIdx.x; item < a.n_items; item += gridDim.x) {
      const Item it = item_of(item);
      if (!it.real) continue;
      float d[128];
      for (int c = 0; c < n_chunks; ++c, ++cc) {
        const int s = cc % STAGES, round = cc / STAGES;
        mbar_wait(bar_full + 8 * s, round & 1);
        const uint32_t st = sbase + s * STAGE_BYTES;
        const uint32_t a_hi = st + wg * 64 * ROW_BYTES, a_lo = st + A_BOX + wg * 64 * ROW_BYTES;
        const uint32_t b_hi = st + 2 * A_BOX, b_lo = st + 2 * A_BOX + B_BOX;
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < KC / 16; ++ks) {
          const uint32_t adv = ks * 32;  // 32 bytes per K step inside the 128-byte swizzle row
          wgmma_ss_f16_n256(d, desc_sw128(a_lo + adv), desc_sw128(b_hi + adv), (c > 0 || ks > 0) ? 1u : 0u);
          wgmma_ss_f16_n256(d, desc_sw128(a_hi + adv), desc_sw128(b_lo + adv), 1u);
          wgmma_ss_f16_n256(d, desc_sw128(a_hi + adv), desc_sw128(b_hi + adv), 1u);
        }
        wgmma_commit();
        if (c > 0) {  // the previous chunk's MMAs are complete: its stage goes back to the producer
          wgmma_wait<1>();
          if ((tid & 127) == 0) mbar_arrive(bar_empty + 8 * ((cc - 1) % STAGES));
        }
      }
      wgmma_wait<0>();
      if ((tid & 127) == 0) mbar_arrive(bar_empty + 8 * ((cc - 1) % STAGES));
#pragma unroll
      for (int i = 0; i < 128; ++i) fence_reg(d[i]);
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        const int r = r0 + 8 * hr;
        const long row = (long)it.tile * TILE + r;
        const float* xk = nullptr;
        if (FIRST) {
          // xk is stored per job and row-blocked, the job's blocks from tile_base[job] + job * xk_pad: window tj * 128 + r reads x row
          // tj * 128 + min(r, rem - 1) + t of the job (the last tile's padding rows repeat its last window), i.e. row xr of block
          // tile + job * xk_pad
          const int xr = min(r, it.rem - 1) + a.t;
          xk = a.xk + (((long)it.tile + (long)it.job * a.xk_pad + (xr >> 7)) * (4 * u) + it.ub * NCOL) * TILE + (xr & (TILE - 1));
        }
        const float* bias = FIRST ? nullptr : a.bias + (long)it.slot * 4 * u + it.ub * NCOL;
        float* ccol = a.c + ((long)it.tile * u + it.ub * UB) * TILE + r;  // unit j of this window: ccol[j * TILE]
        __half2* hh = reinterpret_cast<__half2*>(a.h_out_hi + row * u + it.ub * UB);
        __half2* hl = reinterpret_cast<__half2*>(a.h_out_lo + row * u + it.ub * UB);
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          float hv[2];
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int unit = 8 * jj + 2 * t + e;
            float z[4];
#pragma unroll
            for (int G = 0; G < 4; ++G) z[G] = d[4 * (8 * G + jj) + 2 * hr + e] + (FIRST ? __ldg(xk + (G * UB + unit) * TILE) : __ldg(bias + G * UB + unit));
            const float cp = a.t == 0 ? 0.f : ccol[unit * TILE];
            float cn;
            if (TANH) {
              tanh_cell(z[0], z[1], z[2], z[3], cp, cn, hv[e]);
            } else {
              const float ig = sigm(z[0]), fg = sigm(z[1]), gg = gb::apply_act(a.act, z[2]), og = sigm(z[3]);
              cn = fmaf(fg, cp, ig * gg);
              hv[e] = og * gb::apply_act(a.act, cn);
            }
            ccol[unit * TILE] = cn;
          }
          // FP16 pair h = h1 + h2 (low half = even unit)
          const __half2 p1 = __floats2half2_rn(hv[0], hv[1]);
          const float2 f1 = __half22float2(p1);
          hh[4 * jj + t] = p1;
          hl[4 * jj + t] = __floats2half2_rn(hv[0] - f1.x, hv[1] - f1.y);
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ preparation kernels (fp32 CUDA cores)
// reordered gate column n' = ub*256 + g*64 + j  <->  keras column g*u + ub*64 + j
// Layer widths are padded to multiples of 64 inside this kernel family (zero weights and biases keep the padded units at
// c = h = 0 for all t), so any stack runs on the tensor cores; u below is the REAL width, -1 marks a padded unit.
__device__ __forceinline__ int keras_col(int np, int u) {
  const int ub = np >> 8, g = (np >> 6) & 3, j = np & 63, unit = ub * UB + j;
  return unit < u ? g * u + unit : -1;
}

// weight images of one layer: rows n' (4u per slot), K contiguous: [below part padded to 64 | own part], FP16 pair; slots from slot0
__global__ void lstm_tc_weights_kernel(const float* __restrict__ params, long pstride, long kofs, int in, int u, int up, int kp_below, int kp,
                                       int use_below, int slot0, __half* __restrict__ w_hi, __half* __restrict__ w_lo, float* __restrict__ bias) {
  const int slot = slot0 + blockIdx.y;
  const float* P = params + (long)slot * pstride + kofs;  // kernel [in][4u], recurrent [u][4u], bias [4u]  (real widths)
  const int u4 = 4 * u, up4 = 4 * up;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < (long)up4 * kp; i += (long)gridDim.x * blockDim.x) {
    const int np = (int)(i / kp), k = (int)(i - (long)np * kp);
    const int col = keras_col(np, u);
    float v = 0.f;
    if (col >= 0) {
      if (k < kp_below) {
        if (use_below && k < in) v = P[(long)k * u4 + col];
      } else if (k - kp_below < u) {
        v = P[(long)(in + k - kp_below) * u4 + col];
      }
    }
    const __half h = __float2half_rn(v);
    w_hi[((long)slot * up4 + np) * kp + k] = h;
    w_lo[((long)slot * up4 + np) * kp + k] = __float2half_rn(v - __half2float(h));
  }
  if (blockIdx.x == 0)
    for (int np = threadIdx.x; np < up4; np += blockDim.x) {
      const int col = keras_col(np, u);
      bias[(long)slot * up4 + np] = col >= 0 ? P[(long)(in + u) * u4 + col] : 0.f;
    }
}

// Window tiles are flat: job j owns tiles [tile_base[j], tile_base[j + 1]), ceil(n_rows / 128) of them (the uniform entry gives
// every job max_windows' count).  The record of each tile lets the step and head kernels find an item's job with one load.
__global__ void lstm_tc_uniform_tiles_kernel(int n_jobs, int tiles_per_job, int32_t* __restrict__ tile_base) {
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j <= n_jobs; j += gridDim.x * blockDim.x) tile_base[j] = j * tiles_per_job;
}

__global__ void lstm_tc_tiles_kernel(const gb_job* __restrict__ jobs, int n_jobs, const int32_t* __restrict__ tile_base, int n_tiles, int4* __restrict__ tiles) {
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < n_tiles; t += gridDim.x * blockDim.x) {
    int lo = 0, hi = n_jobs - 1;  // the last job whose first tile is <= t: a job without windows shares its first tile with the next job
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (__ldg(tile_base + mid) <= t) lo = mid; else hi = mid - 1;
    }
    const int tj = t - __ldg(tile_base + lo);
    const int2 sn = __ldg(reinterpret_cast<const int2*>(jobs + lo));  // slot, n_rows
    tiles[t] = tj < 0 ? make_int4(sn.x, 0, lo, 0) : make_int4(sn.x, (int)max(0L, sn.y - (long)tj * TILE), lo, tj);  // a tile before job 0's first holds no window
  }
}

// layer 0 input projection per x row of a job: xk[block][n'][r] = x[x_row + r] . K0[:, col(n')] + b0[col(n')] with the job's slot;
// grid (ceil(rows/32), 4u/64, jobs from job0).  Job j writes its n_rows + lookback - 1 rows into the blocks from tile_base[j] + j * xk_pad
// (never past the next job's first block); a job without windows reads and writes nothing, wherever its x_row points.
__global__ void __launch_bounds__(256) lstm_tc_xk_kernel(const gb_job* __restrict__ jobs, int job0, const int32_t* __restrict__ tile_base, int n_tiles,
                                                         const float* __restrict__ x, int F, int u, int up, int lookback, const float* __restrict__ params,
                                                         long pstride, int xk_pad, float* __restrict__ xk) {
  const int job_id = job0 + blockIdx.z;
  const gb_job job = jobs[job_id];
  const int tb0 = __ldg(tile_base + job_id), tb1 = __ldg(tile_base + job_id + 1);
  if (tb0 < 0 || tb1 < tb0 || tb1 > n_tiles) return;
  const int n_x = job.n_rows == 0 ? 0 : (int)min((long)job.n_rows + lookback - 1, (long)(tb1 - tb0 + xk_pad) * TILE);  // x rows this job's windows touch
  const int r0 = blockIdx.x * 32;
  if (r0 >= n_x) return;
  const float* P = params + (long)job.slot * pstride;  // layer 0: kernel [F][4u] first
  const int u4 = 4 * u, c0 = blockIdx.y * 64;
  __shared__ float sA[32][33];
  __shared__ float sW[32][65];
  const int tid = threadIdx.x, col = tid & 63, rg = tid >> 6;
  const int kc = keras_col(c0 + col, u);
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
  for (int k0 = 0; k0 < F; k0 += 32) {
    for (int i = tid; i < 32 * 32; i += 256) {
      const int b = i >> 5, k = k0 + (i & 31);
      sA[b][i & 31] = (r0 + b < n_x && k < F) ? __ldg(x + (job.x_row + r0 + b) * (long)F + k) : 0.f;
    }
    for (int i = tid; i < 32 * 64; i += 256) {
      const int kk = i >> 6, c = i & 63, k = k0 + kk;
      const int kcol = keras_col(c0 + c, u);
      sW[kk][c] = (k < F && kcol >= 0) ? __ldg(P + (long)k * u4 + kcol) : 0.f;
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
  const float b = kc >= 0 ? __ldg(P + (long)(F + u) * u4 + kc) : 0.f;
  // out: the job's rows, row-blocked [row / 128][4 * up][128]; staged through shared memory so that lanes run along rows (128-byte segments)
#pragma unroll
  for (int i = 0; i < 8; ++i) sW[rg + 4 * i][col] = acc[i] + b;  // sW reused as [32 rows][64 columns]
  __syncthreads();
  float* xj = xk + ((long)tb0 + (long)job_id * xk_pad) * (4L * up) * TILE;
  for (int i = tid; i < 64 * 32; i += 256) {
    const int c = i >> 5, rr = i & 31, r = r0 + rr;
    if (r < n_x) xj[((r >> 7) * (long)(4 * up) + c0 + c) * TILE + (r & (TILE - 1))] = sW[rr][c];
  }
}

// Dense head on the last layer's final h: out[w][o] = act(sum_k h[w][k] Wd[k][o] + bd[o]); one CTA per flat window tile
__global__ void __launch_bounds__(128) lstm_tc_head_kernel(const gb_job* __restrict__ jobs, const int4* __restrict__ tiles, const __half* __restrict__ h_hi,
                                                           const __half* __restrict__ h_lo, int u, int up, int n_out, int out_act,
                                                           const float* __restrict__ params, long pstride, long dofs, float* __restrict__ out) {
  const int4 rec = tiles[blockIdx.x];  // slot, windows of the job from this tile on, job, tile within the job
  if ((int)threadIdx.x >= rec.y) return;
  const int w = rec.w * TILE + threadIdx.x;
  const long row = (long)blockIdx.x * TILE + threadIdx.x;
  const long out_row = jobs[rec.z].out_row;
  const float* Wd = params + (long)rec.x * pstride + dofs;
  const float* bd = Wd + (long)u * n_out;
  for (int o = 0; o < n_out; ++o) {
    float acc = __ldg(bd + o);
    for (int k = 0; k < u; ++k) acc = fmaf(__half2float(h_hi[row * up + k]) + __half2float(h_lo[row * up + k]), __ldg(Wd + (long)k * n_out + o), acc);
    out[(out_row + w) * (long)n_out + o] = gb::apply_act(out_act, acc);
  }
}

// [rows][cols] FP16 row-major, box = 64 columns x box_rows rows, SWIZZLE_128B
int make_map_f16(CUtensorMap* map, const void* base, long rows, long cols, int box_rows) {
  const CUresult r = encode_map_2d(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, sizeof(__half), base, rows, cols, KC, box_rows);
  GB_REQUIRE(r != CUDA_ERROR_NOT_FOUND, GB_E_CUDA, "cuTensorMapEncodeTiled is not available from the driver");
  GB_REQUIRE(r == CUDA_SUCCESS, GB_E_CUDA, "cuTensorMapEncodeTiled (fp16) failed with CUresult %d", (int)r);
  return GB_OK;
}

struct Plan {
  int nl, F, n_out, L;
  int u[GB_MAX_LAYERS], ur[GB_MAX_LAYERS], in[GB_MAX_LAYERS], kp_below[GB_MAX_LAYERS], kp[GB_MAX_LAYERS];  // u: padded to 64, ur / in: real widths
  long kofs[GB_MAX_LAYERS], dofs;
  int xk_pad;  // 128-row xk blocks each job has beyond its window tiles: its windows touch n_rows + lookback - 1 x rows
  // workspace offsets (bytes)
  size_t w_hi[GB_MAX_LAYERS], w_lo[GB_MAX_LAYERS], bias[GB_MAX_LAYERS], h_hi[GB_MAX_LAYERS][2], h_lo[GB_MAX_LAYERS][2], c[GB_MAX_LAYERS], xk, total;
  size_t tile_base, tiles;  // the uniform entry's tile table [n_jobs + 1] and the tile records [n_tiles]
  size_t state_begin, state_end;
};

size_t align256(size_t v) { return (v + 255) / 256 * 256; }

// Sizes follow the flat tiles: the recurrent state holds n_tiles * 128 rows, xk n_tiles + n_jobs * xk_pad blocks.
void make_plan(const gb_lstmnet* net, int n_slots, int n_jobs, long n_tiles, Plan* p) {
  p->nl = net->n_layers; p->F = net->n_features; p->n_out = net->n_features_out; p->L = net->lookback;
  const long rows = n_tiles * TILE;
  p->xk_pad = (p->L - 1 + TILE - 1) / TILE;  // ceil((n + L - 1) / 128) <= ceil(n / 128) + ceil((L - 1) / 128)
  long pofs = 0;
  int in = net->n_features;
  size_t ofs = 0;
  for (int l = 0; l < p->nl; ++l) {
    const int ur = net->units[l], u = gb::round_up(ur, UB);
    p->u[l] = u; p->ur[l] = ur; p->in[l] = in;
    p->kofs[l] = pofs;
    pofs += 4L * ur * (in + ur + 1);
    p->kp_below[l] = l == 0 ? 0 : gb::round_up(in, UB);  // = the padded width of the layer below
    p->kp[l] = p->kp_below[l] + u;
    p->w_hi[l] = ofs; ofs = align256(ofs + (size_t)n_slots * 4 * u * p->kp[l] * sizeof(__half));
    p->w_lo[l] = ofs; ofs = align256(ofs + (size_t)n_slots * 4 * u * p->kp[l] * sizeof(__half));
    p->bias[l] = ofs; ofs = align256(ofs + (size_t)n_slots * 4 * u * sizeof(float));
    in = ur;
  }
  p->dofs = pofs;
  p->tile_base = ofs; ofs = align256(ofs + (size_t)(n_jobs + 1) * sizeof(int32_t));
  p->tiles = ofs; ofs = align256(ofs + (size_t)n_tiles * sizeof(int4));
  p->xk = ofs; ofs = align256(ofs + (size_t)(n_tiles + (long)n_jobs * p->xk_pad) * TILE * 4 * p->u[0] * sizeof(float));
  p->state_begin = ofs;
  for (int l = 0; l < p->nl; ++l) {
    const size_t hb = (size_t)rows * p->u[l] * sizeof(__half);
    for (int b = 0; b < 2; ++b) {
      p->h_hi[l][b] = ofs; ofs = align256(ofs + hb);
      p->h_lo[l][b] = ofs; ofs = align256(ofs + hb);
    }
    p->c[l] = ofs; ofs = align256(ofs + (size_t)rows * p->u[l] * sizeof(float));
  }
  p->state_end = ofs;
  p->total = ofs;
}

constexpr long MAX_TILES = (1L << 31) / (512 / UB) - 1;  // work items (tile, unit block) are counted in int

// Host-side checks shared by both entries; n_tiles as a long so that a uniform layout too large to count is refused, not wrapped.
int check_sizes(int32_t n_slots, int32_t n_jobs, long n_tiles, int32_t max_windows) {
  GB_REQUIRE(n_jobs >= 0 && max_windows >= 0 && n_slots >= 1 && n_tiles >= 0, GB_E_ARG, "bad n_jobs=%d / max_windows=%d / n_slots=%d / n_tiles=%ld",
             n_jobs, max_windows, n_slots, n_tiles);
  const long tiles_per_job = ((long)max_windows + TILE - 1) / TILE;
  GB_REQUIRE(n_tiles <= (long)n_jobs * tiles_per_job, GB_E_SHAPE, "n_tiles=%ld exceeds n_jobs * ceil(max_windows / 128) = %ld", n_tiles,
             (long)n_jobs * tiles_per_job);
  GB_REQUIRE(n_tiles <= MAX_TILES, GB_E_SHAPE, "n_tiles=%ld exceeds %ld window tiles per launch", n_tiles, MAX_TILES);
  return GB_OK;
}

// tile_base == nullptr: the uniform layout, every job ceil(max_windows / 128) tiles, its table written into the workspace
int infer_tc(const gb_lstmnet* net, const float* params, int32_t n_slots, const gb_job* jobs, int32_t n_jobs, const int32_t* tile_base, int n_tiles,
             int32_t max_windows, const float* x, float* out_model, void* workspace, cudaStream_t st) {
  int rc;
  GB_REQUIRE(gb::aligned16(workspace), GB_E_ALIGN, "workspace must be 16-byte aligned");
  if (n_jobs == 0 || n_tiles == 0 || max_windows == 0) return GB_OK;
  const long rows = (long)n_tiles * TILE;
  Plan p;
  make_plan(net, n_slots, n_jobs, n_tiles, &p);
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  const long pstride = (long)gb_lstm_param_stride(net);
  constexpr int GRID_YZ = 65535;  // gridDim.y / z carry slots and jobs: larger fleets go out as several launches

  // ---- the tile table and the per-tile records
  if (tile_base == nullptr) {
    int32_t* tb = reinterpret_cast<int32_t*>(ws + p.tile_base);
    lstm_tc_uniform_tiles_kernel<<<(n_jobs + 256) / 256, 256, 0, st>>>(n_jobs, (max_windows + TILE - 1) / TILE, tb);
    tile_base = tb;
  }
  int4* tiles = reinterpret_cast<int4*>(ws + p.tiles);
  lstm_tc_tiles_kernel<<<min((n_tiles + 255) / 256, 4096), 256, 0, st>>>(jobs, n_jobs, tile_base, n_tiles, tiles);

  // ---- operands that do not depend on the timestep
  for (int l = 0; l < p.nl; ++l)
    for (int s0 = 0; s0 < n_slots; s0 += GRID_YZ)
      lstm_tc_weights_kernel<<<dim3(64, min(n_slots - s0, GRID_YZ)), 256, 0, st>>>(params, pstride, p.kofs[l], p.in[l], p.ur[l], p.u[l], p.kp_below[l],
                                                                                  p.kp[l], l > 0, s0, reinterpret_cast<__half*>(ws + p.w_hi[l]),
                                                                                  reinterpret_cast<__half*>(ws + p.w_lo[l]), reinterpret_cast<float*>(ws + p.bias[l]));
  const int xr_max = max_windows + p.L - 1;
  for (int j0 = 0; j0 < n_jobs; j0 += GRID_YZ)
    lstm_tc_xk_kernel<<<dim3((xr_max + 31) / 32, 4 * p.u[0] / 64, min(n_jobs - j0, GRID_YZ)), 256, 0, st>>>(
        jobs, j0, tile_base, n_tiles, x, p.F, p.ur[0], p.u[0], p.L, params, pstride, p.xk_pad, reinterpret_cast<float*>(ws + p.xk));
  GB_CUDA_CHECK(cudaMemsetAsync(ws + p.state_begin, 0, p.state_end - p.state_begin, st));
  GB_CUDA_CHECK(cudaGetLastError());

  CUtensorMap m_h[GB_MAX_LAYERS][2][2], m_w[GB_MAX_LAYERS][2];
  for (int l = 0; l < p.nl; ++l) {
    for (int b = 0; b < 2; ++b) {
      if ((rc = make_map_f16(&m_h[l][b][0], ws + p.h_hi[l][b], rows, p.u[l], TILE)) != GB_OK) return rc;
      if ((rc = make_map_f16(&m_h[l][b][1], ws + p.h_lo[l][b], rows, p.u[l], TILE)) != GB_OK) return rc;
    }
    if ((rc = make_map_f16(&m_w[l][0], ws + p.w_hi[l], (long)n_slots * 4 * p.u[l], p.kp[l], NCOL)) != GB_OK) return rc;
    if ((rc = make_map_f16(&m_w[l][1], ws + p.w_lo[l], (long)n_slots * 4 * p.u[l], p.kp[l], NCOL)) != GB_OK) return rc;
  }
  const size_t smem = (size_t)STAGES * STAGE_BYTES + 1024;  // + alignment slack of the 1 KB aligned ring
  int dev = 0, sms = 132;
  GB_CUDA_CHECK(cudaGetDevice(&dev));
  GB_CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  using StepKernel = void (*)(const TcLayerArgs, const CUtensorMap, const CUtensorMap, const CUtensorMap, const CUtensorMap, const CUtensorMap, const CUtensorMap);
  const StepKernel kernels[2][2] = {{lstm_tc_step_kernel<false, false>, lstm_tc_step_kernel<false, true>},
                                    {lstm_tc_step_kernel<true, false>, lstm_tc_step_kernel<true, true>}};
  for (int f = 0; f < 2; ++f)
    for (int q = 0; q < 2; ++q) GB_CUDA_CHECK(cudaFuncSetAttribute(kernels[f][q], cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));

  // ---- the recurrence: h of (layer, t) is written to buffer t & 1 and read from buffer (t - 1) & 1 (zero at t = 0)
  for (int t = 0; t < p.L; ++t) {
    const int wr = t & 1, rd = wr ^ 1;
    for (int l = 0; l < p.nl; ++l) {
      TcLayerArgs a{};
      a.u = p.u[l]; a.kc_below = p.kp_below[l] / KC; a.kc_own = p.u[l] / KC; a.act = net->act[l];
      a.t = t; a.tiles = tiles;
      a.bias = reinterpret_cast<const float*>(ws + p.bias[l]);
      a.xk = reinterpret_cast<const float*>(ws + p.xk); a.xk_pad = p.xk_pad;
      a.c = reinterpret_cast<float*>(ws + p.c[l]);
      a.h_out_hi = reinterpret_cast<__half*>(ws + p.h_hi[l][wr]);
      a.h_out_lo = reinterpret_cast<__half*>(ws + p.h_lo[l][wr]);
      const int lb = l > 0 ? l - 1 : 0;
      a.n_items = n_tiles * (p.u[l] / UB);
      const int grid = a.n_items < sms ? a.n_items : sms;
      kernels[l == 0][net->act[l] == GB_ACT_TANH]<<<grid, NTHREADS, smem, st>>>(a, m_h[lb][wr][0], m_h[lb][wr][1], m_h[l][rd][0], m_h[l][rd][1],
                                                                              m_w[l][0], m_w[l][1]);
      GB_CUDA_CHECK(cudaGetLastError());
    }
  }
  const int top = p.nl - 1, fin = (p.L - 1) & 1;
  lstm_tc_head_kernel<<<n_tiles, TILE, 0, st>>>(jobs, tiles, reinterpret_cast<const __half*>(ws + p.h_hi[top][fin]),
                                                reinterpret_cast<const __half*>(ws + p.h_lo[top][fin]), p.ur[top], p.u[top], p.n_out, net->out_act, params,
                                                pstride, p.dofs, out_model);
  GB_CUDA_CHECK(cudaGetLastError());
  return GB_OK;
}

}  // namespace

extern "C" int gb_lstm_tc_supported(const gb_lstmnet* net) {
  GB_REQUIRE(net != nullptr, GB_E_ARG, "net is NULL");
  GB_REQUIRE(net->n_layers >= 1 && net->n_layers <= GB_MAX_LAYERS, GB_E_SHAPE, "n_layers=%d outside [1,%d]", net->n_layers, GB_MAX_LAYERS);
  for (int l = 0; l < net->n_layers; ++l)
    GB_REQUIRE(net->units[l] >= 1 && net->units[l] <= 512, GB_E_SHAPE, "tensor-core LSTM variant covers layer widths 1..512, units[%d]=%d", l, net->units[l]);
  GB_REQUIRE(net->n_features >= 1 && net->n_features <= 512 && net->n_features_out >= 1 && net->n_features_out <= 512, GB_E_SHAPE, "bad feature counts");
  GB_REQUIRE(net->lookback >= 1, GB_E_ARG, "lookback=%d must be >= 1", net->lookback);
  for (int l = 0; l < net->n_layers; ++l)  // h is carried as an FP16 pair: only cells with |h| < 1
    GB_REQUIRE(net->act[l] == GB_ACT_TANH || net->act[l] == GB_ACT_SIGMOID, GB_E_SHAPE,
               "tensor-core LSTM variant covers tanh and sigmoid cells (a relu or linear cell's h overflows FP16), act[%d]=%d", l, net->act[l]);
  return GB_OK;
}

// x_rows: rows of the x array (not needed for the size: each job's input projection covers its own n_rows + lookback - 1 rows)
extern "C" size_t gb_lstm_tc_workspace_bytes(const gb_lstmnet* net, int32_t n_slots, int32_t n_jobs, int32_t max_windows, int64_t /*x_rows*/) {
  if (gb_lstm_tc_supported(net) != GB_OK || n_jobs < 0 || max_windows < 0 || n_slots < 0) return 0;
  Plan p;
  make_plan(net, n_slots, n_jobs, (long)n_jobs * ((max_windows + TILE - 1) / TILE), &p);
  return p.total;
}

extern "C" size_t gb_lstm_tc_ragged_workspace_bytes(const gb_lstmnet* net, int32_t n_slots, int32_t n_jobs, int32_t n_tiles, int32_t max_windows) {
  const long tiles_per_job = ((long)max_windows + TILE - 1) / TILE;
  if (gb_lstm_tc_supported(net) != GB_OK || n_slots < 0 || n_jobs < 0 || max_windows < 0 || n_tiles < 0 || n_tiles > n_jobs * tiles_per_job ||
      n_tiles > MAX_TILES)
    return 0;
  Plan p;
  make_plan(net, n_slots, n_jobs, n_tiles, &p);
  return p.total;
}

extern "C" int gb_lstm_infer_tc(const gb_lstmnet* net, const float* params, int32_t n_slots, const gb_job* jobs, int32_t n_jobs, int32_t max_windows,
                                const float* x, int64_t x_rows, float* out_model, void* workspace, void* stream) {
  int rc = gb_lstm_tc_supported(net);
  if (rc != GB_OK) return rc;
  GB_REQUIRE(params && jobs && x && out_model && workspace, GB_E_ARG, "params/jobs/x/out_model/workspace must be non-NULL");
  GB_REQUIRE(n_jobs >= 0 && max_windows >= 0 && n_slots >= 1 && x_rows >= 1, GB_E_ARG, "bad n_jobs/max_windows/n_slots/x_rows");
  const long n_tiles = (long)n_jobs * ((max_windows + TILE - 1) / TILE);
  if ((rc = check_sizes(n_slots, n_jobs, n_tiles, max_windows)) != GB_OK) return rc;
  return infer_tc(net, params, n_slots, jobs, n_jobs, nullptr, (int)n_tiles, max_windows, x, out_model, workspace, (cudaStream_t)stream);
}

extern "C" int gb_lstm_infer_tc_ragged(const gb_lstmnet* net, const float* params, int32_t n_slots, const gb_job* jobs, int32_t n_jobs,
                                       const int32_t* tile_base, int32_t n_tiles, int32_t max_windows, const float* x, int64_t x_rows,
                                       float* out_model, void* workspace, void* stream) {
  int rc = gb_lstm_tc_supported(net);
  if (rc != GB_OK) return rc;
  GB_REQUIRE(params && jobs && tile_base && x && out_model && workspace, GB_E_ARG, "params/jobs/tile_base/x/out_model/workspace must be non-NULL");
  GB_REQUIRE(x_rows >= 1, GB_E_ARG, "x_rows=%lld must be >= 1", (long long)x_rows);
  if ((rc = check_sizes(n_slots, n_jobs, n_tiles, max_windows)) != GB_OK) return rc;
  return infer_tc(net, params, n_slots, jobs, n_jobs, tile_base, n_tiles, max_windows, x, out_model, workspace, (cudaStream_t)stream);
}
