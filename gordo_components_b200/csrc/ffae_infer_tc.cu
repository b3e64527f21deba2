// K1+K4, variant 2: fused Dense-stack forward + anomaly score on the Hopper tensor cores (warpgroup MMA, wgmma).
//
// Covers autoencoders of 24..64 tags (multiples of 4; narrower rows ride in zero-padded columns) with hidden widths <= 64
// (feedforward_hourglass(64) = 64-53-43-32-32-43-53-64 is the BASELINE workload).  The path is bound by HBM traffic
// (1 548 algorithmic bytes and 30 236 FLOP per window): fp32 CUDA cores would be the limit, the tensor cores are not.
//
// Numerics: 1e-4 parity with the float32 reference forbids plain TF32/FP16 (2^-11 per operand), so operands are split.
// Layer 0 (x is raw data of any magnitude):
//        D  =  A_hi*W_hi                              (tf32, A_hi = A truncated to TF32, W_hi = W rounded to TF32)
//           +  bf16(A - A_hi)*bf16(W_hi)  +  bf16(A)*bf16(W - W_hi)   (bf16: the 2^-11-sized corrections need only 8 bits)
// Layers >= 1 (A = tanh(.) in [-1, 1], so FP16 cannot overflow): A = a1 + a2, W = w1 + w2 with a1 = fp16(A),
// a2 = fp16(A - a1) and likewise for W (22 significant bits each):
//        D  =  a2*w1  +  a1*w2  +  a1*w1          (f16, products exact in the fp32 accumulator, dropped a2*w2 ~ 2^-22)
// Accumulation is fp32; error against the float64 oracle ~2e-6 absolute.
//
// One persistent CTA per SM, NWG warpgroups.  Per work item (a range of one job's rows) the slot's weights are split and
// laid out once in shared memory as K-major wgmma B operands.  A warpgroup owns a 64-row tile at a time, one thread per
// (row pair, column pair) as the wgmma fragments lay it out: x is read from a shared-memory tile into the A fragment of
// layer 0, and every layer's accumulator becomes the next layer's A fragment in registers (bias, tanh, FP16 split), so
// activations never leave the register file.  The output layer's accumulator is scored against y, read from a second
// shared-memory tile in the same fragment layout.  Each warpgroup owns one x and one y tile buffer, filled by TMA: the next
// tile's x is requested as soon as layer 0 has read the current one, so it loads behind a whole tile of MMAs.  Every per-tag
// output goes out through shared memory: each warp writes its 16 rows x 32 columns of an array into a 2 KB box and one lane
// hands the box to a TMA store, so the writes reach HBM as whole lines and the warp moves on while they drain.  The warp's
// two boxes are its two slices of the y tile (free once y is in registers), so y of a tile is requested only after layer 0 of
// that tile, once the previous tile's stores have read their boxes; it loads behind layers 1 ..  The warpgroups of an SM
// overlap one another's tensor-core waits.
//
// Reference arithmetic replaced: keras Dense under Model.predict (gordo/machine/model/models.py:289-300) and
// DiffBasedAnomalyDetector.anomaly (gordo/machine/model/anomaly/diff.py:350-385, 420-444).
#include <atomic>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include "gb_common.cuh"
#include "gb_sm90.cuh"

namespace {

using namespace gb::sm90;

constexpr int TILE = 64;  // rows per warpgroup tile (wgmma M)
constexpr int NWG_MAX = 3;  // warpgroups per CTA (float64 x tiles of a stack whose weights leave no room for three: 2)
constexpr int MAXL = 8;
constexpr int W = 64;  // widest feature / hidden width
// x / y tiles in shared memory: 64 rows x 64 columns of fp32 as two TMA boxes of 32 columns (128-byte rows, SWIZZLE_128B).
// float64 x (the input-scaler mode) is four boxes of 16 columns: the same 128-byte rows, twice the bytes per tile.
constexpr int BOX_COLS = 32;
constexpr int BOX_COLS_X64 = 16;
constexpr int BOX_BYTES = TILE * BOX_COLS * 4;
constexpr int TILE_BYTES = 2 * BOX_BYTES;
// per warpgroup: one x and one y tile
__host__ __device__ constexpr int x_tile_bytes(bool x64) { return x64 ? 2 * TILE_BYTES : TILE_BYTES; }
__host__ __device__ constexpr int stage_bytes(bool x64, int nwg) { return (x_tile_bytes(x64) + TILE_BYTES) * nwg; }
// output staging: a warp's 16 rows x 32 columns of one array (rows 16 wq .. of a SWIZZLE_128B box: a 1024-aligned slice)
constexpr int OBOX_ROWS = 16;
constexpr int OBOX_BYTES = OBOX_ROWS * BOX_COLS * 4;
// parameter loads per thread and layer when the weights are restaged: a layer's kernel and bias are one batch of loads
__host__ __device__ constexpr int restage_batch(int nthreads) { return (W * W + W + nthreads - 1) / nthreads; }
static_assert(restage_batch(128 * NWG_MAX) == 11, "three warpgroups restage a layer in 11 loads per thread");

struct TcArgs {
  CUtensorMap tm_x, tm_y;  // x and y as [n_x_rows][T], boxes of BOX_COLS x TILE, zeros outside (tm_y unused without y)
  CUtensorMap tm_o[4];     // model output, tag-anomaly-unscaled, -scaled, confidence as [n_out_rows][T], boxes of BOX_COLS x OBOX_ROWS
  int T;  // tags per row of x / y / every per-tag output (row pitch); <= W, multiple of 4
  int L;  // layers
  int N[MAXL], Np[MAXL], k16[MAXL];                  // Np = N rounded up to 16 (wgmma N), k16 = K steps of 16
  int img0_ofs[MAXL], img1_ofs[MAXL], img2_ofs[MAXL];  // byte offsets into dynamic smem of the weight images
  int bias_ofs[MAXL];
  int pofs[MAXL];  // float offsets of W_l in the canonical parameter vector
  int K[MAXL];
  int w_bytes;  // bytes of the weight+bias region (zero-filled before staging)
  int vec_ofs;
  int stage_ofs;  // x / y tile buffers: the first 1024-byte boundary at or after this offset (SWIZZLE_128B boxes)
  int n_jobs, tiles_per_job;
  long pstride;
  const float* params;
  const gb_job* jobs;
  const float *y, *scale, *feat_thr, *agg_thr;  // (x and y are read through tm_x / tm_y; y != nullptr says whether it is given)
  float *o_model, *o_ts, *o_tu, *o_conf, *o_tots, *o_totu, *o_totconf;
  unsigned int* work_ctr;  // global tile counter of this launch (zeroed by the launcher, stream-ordered)
  // float64 x only: x' = (float)(x * x_scale[slot][c] + x_offset[slot][c]), the slot's pair staged at xab_ofs as double [2][W]
  const double *x_scale, *x_offset;
  int xab_ofs;
  long n_x_rows;
};

// tanh(x) = 1 - 2/(1 + 2^(2x*log2 e)); absolute error ~2e-7 (ex2.approx / rcp.approx are ~1-2 ulp), exact limits at +-inf.
// The argument arrives pre-scaled: t = (z + b) * 2*log2(e) is formed as fma(z, TANH_ARG_SCALE, b*TANH_ARG_SCALE).
constexpr float TANH_ARG_SCALE = 2.8853900817779268f;
__device__ __forceinline__ float tanh_from_scaled(float t) {
  float e, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(t));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(e + 1.0f));
  return fmaf(-2.0f, r, 1.0f);
}

__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  const __nv_bfloat162 p = __floats2bfloat162_rn(lo, hi);  // low half = even k (the order the MMA expects)
  return *reinterpret_cast<const uint32_t*>(&p);
}
__device__ __forceinline__ float trunc_tf32(float v) { return __uint_as_float(__float_as_uint(v) & 0xffffe000u); }
// FP16 pair of two activations: w1 = fp16(a), w2 = fp16(a - w1)
__device__ __forceinline__ void split_f16(float a0, float a1, uint32_t& w1, uint32_t& w2) {
  const __half2 h = __floats2half2_rn(a0, a1);
  const float2 f = __half22float2(h);
  const __half2 r = __floats2half2_rn(a0 - f.x, a1 - f.y);
  w1 = *reinterpret_cast<const uint32_t*>(&h);
  w2 = *reinterpret_cast<const uint32_t*>(&r);
}

// Position of weight row k inside layer 0's TF32 image.  A thread's x registers hold, per 16 columns, the pairs 2t, 2t+1 and
// 2t+8, 2t+9 (the 16-bit A fragment); the TF32 MMA (K = 8) expects columns t and t+4 of each 8.  The sum over K does not
// care about the order, so the TF32 steps take the registers as they are and the weight rows are permuted to match:
// column 8s + 2t + e of the data is row 8s + t + 4e of the image.
__host__ __device__ __forceinline__ int tf32_row(int k) { return (k & ~7) | (((k & 7) >> 1) + 4 * (k & 1)); }

// ---- one layer's MMAs for wgmma width N (the accumulator is d[0 .. N/2))
template <int N>
__device__ __forceinline__ void mma_layer0(float* d, const uint32_t (&xhi)[4][8], const uint32_t (&alo)[4][4], const uint32_t (&abf)[4][4],
                                           uint32_t img0, uint32_t img1, uint32_t img2, int k16) {
  const uint32_t lbo = N * 16, step = 2 * N * 16;
#pragma unroll
  for (int ks = 0; ks < 8; ++ks)  // A_hi * W_hi, first MMA overwrites
    if (ks < 2 * k16) {
      const uint32_t a[4] = {xhi[ks >> 1][4 * (ks & 1) + 0], xhi[ks >> 1][4 * (ks & 1) + 1], xhi[ks >> 1][4 * (ks & 1) + 2], xhi[ks >> 1][4 * (ks & 1) + 3]};
      if (N == 16) wgmma_rs_tf32_n16(d, a, desc_noswizzle(img0 + ks * step, lbo, 128), ks > 0);
      if (N == 32) wgmma_rs_tf32_n32(d, a, desc_noswizzle(img0 + ks * step, lbo, 128), ks > 0);
      if (N == 48) wgmma_rs_tf32_n48(d, a, desc_noswizzle(img0 + ks * step, lbo, 128), ks > 0);
      if (N == 64) wgmma_rs_tf32_n64(d, a, desc_noswizzle(img0 + ks * step, lbo, 128), ks > 0);
    }
#pragma unroll
  for (int ks = 0; ks < 4; ++ks)  // bf16(A_lo) * bf16(W_hi)
    if (ks < k16) {
      if (N == 16) wgmma_rs_bf16_n16(d, alo[ks], desc_noswizzle(img1 + ks * step, lbo, 128), 1);
      if (N == 32) wgmma_rs_bf16_n32(d, alo[ks], desc_noswizzle(img1 + ks * step, lbo, 128), 1);
      if (N == 48) wgmma_rs_bf16_n48(d, alo[ks], desc_noswizzle(img1 + ks * step, lbo, 128), 1);
      if (N == 64) wgmma_rs_bf16_n64(d, alo[ks], desc_noswizzle(img1 + ks * step, lbo, 128), 1);
    }
#pragma unroll
  for (int ks = 0; ks < 4; ++ks)  // bf16(A) * bf16(W_lo)
    if (ks < k16) {
      if (N == 16) wgmma_rs_bf16_n16(d, abf[ks], desc_noswizzle(img2 + ks * step, lbo, 128), 1);
      if (N == 32) wgmma_rs_bf16_n32(d, abf[ks], desc_noswizzle(img2 + ks * step, lbo, 128), 1);
      if (N == 48) wgmma_rs_bf16_n48(d, abf[ks], desc_noswizzle(img2 + ks * step, lbo, 128), 1);
      if (N == 64) wgmma_rs_bf16_n64(d, abf[ks], desc_noswizzle(img2 + ks * step, lbo, 128), 1);
    }
}
template <int N>
__device__ __forceinline__ void mma_f16(float* d, const uint32_t* a, uint64_t desc, uint32_t acc) {
  if (N == 16) wgmma_rs_f16_n16(d, a, desc, acc);
  if (N == 32) wgmma_rs_f16_n32(d, a, desc, acc);
  if (N == 48) wgmma_rs_f16_n48(d, a, desc, acc);
  if (N == 64) wgmma_rs_f16_n64(d, a, desc, acc);
}
template <int N>
__device__ __forceinline__ void mma_hidden(float* d, const uint32_t (&a1)[4][4], const uint32_t (&a2)[4][4], uint32_t img0, uint32_t img1, int k16) {
  const uint32_t lbo = N * 16, step = 2 * N * 16;
#pragma unroll
  for (int ks = 0; ks < 4; ++ks)  // a2 * w1 (first MMA overwrites the accumulator)
    if (ks < k16) mma_f16<N>(d, a2[ks], desc_noswizzle(img0 + ks * step, lbo, 128), ks > 0);
#pragma unroll
  for (int ks = 0; ks < 4; ++ks)  // a1 * w2
    if (ks < k16) mma_f16<N>(d, a1[ks], desc_noswizzle(img1 + ks * step, lbo, 128), 1);
#pragma unroll
  for (int ks = 0; ks < 4; ++ks)  // a1 * w1
    if (ks < k16) mma_f16<N>(d, a1[ks], desc_noswizzle(img0 + ks * step, lbo, 128), 1);
}

// Byte offset inside a staged tile of the float pair (row r, columns col, col + 1), col even.  SWIZZLE_128B stores the 16-byte
// chunk c of a box row r at chunk c ^ (r % 8), so the eight rows g of a warp's fragment access fall in different chunks: each
// 8-byte access of a warp touches every bank exactly twice (two wavefronts, the least for 256 bytes).
// The same inside one box (col < 32); the output staging boxes use it too.
__device__ __forceinline__ int box_ofs(int r, int col) { return r * 128 + (((col >> 2) ^ (r & 7)) << 4) + ((col & 3) << 2); }
__device__ __forceinline__ int tile_ofs(int r, int col) { return (col >> 5) * BOX_BYTES + box_ofs(r, col & 31); }
// ... and of the double pair (row r, columns col, col + 1) in a float64 x tile: one whole 16-byte chunk, boxes of 16 columns
__device__ __forceinline__ int tile_ofs_x64(int r, int col) { return (col >> 4) * BOX_BYTES + r * 128 + ((((col & 15) >> 1) ^ (r & 7)) << 4); }

__device__ __forceinline__ void warpgroup_sync(int wg) { asm volatile("bar.sync %0, 128;" ::"r"(wg + 1) : "memory"); }

__device__ __forceinline__ void fence_acc(float (&d)[32]) {
#pragma unroll
  for (int i = 0; i < 32; ++i) fence_reg(d[i]);
}
// the tensor cores read register A operands asynchronously: they stay allocated until the wait that follows the MMAs
template <int R, int C>
__device__ __forceinline__ void fence_frag(uint32_t (&f)[R][C]) {
#pragma unroll
  for (int i = 0; i < R; ++i)
#pragma unroll
    for (int j = 0; j < C; ++j) fence_reg(f[i][j]);
}

// ------------------------------------------------------------------------------------------------ kernel
// X64: x is float64 and the slot's input scaler is applied as each element is read (a.x_scale / a.x_offset).
template <bool X64, int NWG>
__global__ void __launch_bounds__(128 * NWG, 1) ffae_tc_kernel(const __grid_constant__ TcArgs a) {
  constexpr int NTHREADS = 128 * NWG;
  constexpr int RESTAGE_BATCH = restage_batch(NTHREADS);
  extern __shared__ __align__(1024) uint8_t smem[];
  const int tid = threadIdx.x, lane = tid & 31;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
  const int wg = warp >> 2, wq = warp & 3;  // warpgroup; warp inside it (rows 16 wq ..)
  const int g = lane >> 2, t = lane & 3;    // fragment row / column pair
  const uint32_t sbase = smem_u32(smem);
  const int TP = a.T, L = a.L;
  const bool has_y = a.y != nullptr;
  const bool totals = has_y && (a.o_tots || a.o_totu || a.o_totconf);
  const float inv_w = 1.0f / (float)TP;

  // this warpgroup's x and y tiles, and the mbarriers their TMA loads complete on; thread 0 of the warpgroup issues the loads
  __shared__ __align__(8) unsigned long long s_bar[2 * NWG];
  const uint32_t stage = (sbase + a.stage_ofs + 1023) & ~1023u;
  const uint32_t xbuf = stage + wg * (x_tile_bytes(X64) + TILE_BYTES), ybuf = xbuf + x_tile_bytes(X64);
  const uint8_t* xs = smem + (xbuf - sbase);
  const uint8_t* ys = smem + (ybuf - sbase);
  const uint32_t bar_x = smem_u32(&s_bar[wg]), bar_y = smem_u32(&s_bar[NWG + wg]);
  const bool leader = (tid & 127) == 0;
  uint32_t x_phase = 0, y_phase = 0;
  // this warp's output staging boxes (lane 0 issues their TMA stores)
  const uint32_t obox0 = ybuf + wq * OBOX_BYTES, obox1 = obox0 + BOX_BYTES;
  if (tid == 0) {
    for (int i = 0; i < 2 * NWG; ++i) mbar_init(smem_u32(&s_bar[i]), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }

  // Work distribution.  Tiles are numbered job by job (global tile G = job * tiles_per_job + tile) and handed out from a global
  // counter in contiguous ranges: whole jobs, in order, for most of the launch (a change of job restages the weights), then
  // thirds and sixths of a job for the last ~1.5 jobs per CTA, so that the SMs finish close together.
  __shared__ int s_item[3];   // job, first tile, end tile of the item all threads work on next
  __shared__ int s_range[2];  // thread 0: tiles [g, g_end) of the range it holds
  if (tid == 0) s_range[0] = s_range[1] = 0;
  int cur_slot = -1;

  while (true) {
    if (tid == 0) {
      const int tpj = a.tiles_per_job, g_total = a.n_jobs * tpj;  // (the launcher refuses fleets beyond 2^31 tiles)
      int gg = s_range[0], g_end = s_range[1];
      if (gg >= g_end) {
        const int seen = (int)*reinterpret_cast<volatile unsigned int*>(a.work_ctr);
        const int left = g_total - seen, per_cta = left / (int)gridDim.x;
        int size = per_cta * 2 >= 3 * tpj ? tpj : (per_cta >= tpj / 3 ? (tpj + 2) / 3 : (tpj + 5) / 6);
        if (size < 1) size = 1;
        if (seen % tpj != 0 && size > tpj - seen % tpj) size = tpj - seen % tpj;  // ranges end at job boundaries (a stale `seen` at worst mis-sizes one)
        gg = (int)atomicAdd(a.work_ctr, (unsigned int)size);
        g_end = gg + size < g_total ? gg + size : g_total;
      }
      if (gg >= g_total) {
        s_item[0] = -1;
      } else {
        const int job_id = gg / tpj, tile_begin = gg - job_id * tpj;
        const int tile_end = min(tpj, tile_begin + (g_end - gg));
        s_item[0] = job_id; s_item[1] = tile_begin; s_item[2] = tile_end;
        gg += tile_end - tile_begin;
      }
      s_range[0] = gg; s_range[1] = g_end;
    }
    __syncthreads();
    const int job_id = s_item[0], tile_begin = s_item[1], tile_end = s_item[2];
    if (job_id < 0) break;
    const gb_job job = a.jobs[job_id];
    const int row_begin = tile_begin * TILE;
    if (row_begin >= job.n_rows) {  // uniform across the CTA
      __syncthreads();              // every thread has read s_item before thread 0 writes the next one
      continue;
    }
    const int row_end = min(job.n_rows, tile_end * TILE);
    const int n_tiles = (row_end - row_begin + TILE - 1) / TILE;

    // One 64-row tile of x or y for this warpgroup (thread 0 of the warpgroup).  Columns past T and rows past the end of the array
    // arrive as zeros; rows past the end of the job are its neighbour's rows.  Those rows run through the MMAs like any other (the
    // rows of an MMA are independent) and nothing of them is stored.
    auto load_tile = [&](const CUtensorMap* m, uint32_t buf, uint32_t bar, int tt) {
      const int row = (int)(job.x_row + row_begin + tt * TILE);
      mbar_expect_tx(bar, TILE_BYTES);
      tma_load_2d(buf, m, 0, row, bar);
      tma_load_2d(buf + BOX_BYTES, m, BOX_COLS, row, bar);
    };
    // ... and a float64 x tile: four boxes of 16 columns
    auto load_x64 = [&](int tt) {
      const int row = (int)(job.x_row + row_begin + tt * TILE);
      mbar_expect_tx(bar_x, x_tile_bytes(true));
#pragma unroll
      for (int h = 0; h < 4; ++h) tma_load_2d(xbuf + h * BOX_BYTES, &a.tm_x, BOX_COLS_X64 * h, row, bar_x);
    };
    // the x buffer is free between items (the last tile requested no successor): the first tile loads behind the restage
    if (leader && wg < n_tiles) {
      if constexpr (X64) load_x64(wg);
      else load_tile(&a.tm_x, xbuf, bar_x, wg);
    }

    // ---- stage this slot's weights: split (layer 0: TF32-hi + BF16 hi / lo, others: FP16 pair) as K-major wgmma B operands
    if (job.slot != cur_slot) {
      cur_slot = job.slot;
      const float* P = a.params + (long)job.slot * a.pstride;
      // The restage is bound by the latency of its loads (the SM streams no tiles meanwhile).  A layer's kernel [K][N] and bias
      // [N] (contiguous in the parameter vector, K * N + N <= RESTAGE_BATCH * NTHREADS) are one batch of loads per thread, and the
      // batch of layer l + 1 is requested before layer l is split, so it arrives while that layer is written.  Layer 0's batch
      // and the per-tag vectors are requested ahead of the zero fill.
      float v[RESTAGE_BATCH], vn[RESTAGE_BATCH];
      auto fetch = [&](float (&dst)[RESTAGE_BATCH], int l) {
        const float* Ws = P + a.pofs[l];
        const int n_l = a.K[l] * a.N[l] + a.N[l];
#pragma unroll
        for (int u = 0; u < RESTAGE_BATCH; ++u) {
          const int i = tid + u * NTHREADS;
          dst[u] = i < n_l ? __ldg(Ws + i) : 0.f;
        }
      };
      fetch(v, 0);
      const bool vt = tid < TP;
      const float sc = vt && a.scale ? __ldg(a.scale + (long)job.slot * TP + tid) : 0.f;
      const float ft = vt && a.feat_thr ? __ldg(a.feat_thr + (long)job.slot * TP + tid) : 0.f;
      for (int i = tid; i < a.w_bytes / 16; i += NTHREADS) reinterpret_cast<uint4*>(smem)[i] = make_uint4(0, 0, 0, 0);
      __syncthreads();
      for (int l = 0; l < L; ++l) {
        if (l + 1 < L) fetch(vn, l + 1);
        const int K = a.K[l], N = a.N[l], Np = a.Np[l], KN = K * N;
        const float bscale = (l + 1 < L) ? TANH_ARG_SCALE : 1.0f;  // hidden layers: bias folded into the tanh argument scale
#pragma unroll
        for (int u = 0; u < RESTAGE_BATCH; ++u) {
          const int i = tid + u * NTHREADS;
          if (i >= KN + N) break;
          if (i >= KN) {
            reinterpret_cast<float*>(smem + a.bias_ofs[l])[i - KN] = v[u] * bscale;
            continue;
          }
          const int k = i / N, n = i - k * N;
          const float w = v[u];
          const int i8 = ((k >> 3) * Np + n) * 8 + (k & 7);  // [K/8][Np][8] 16-bit images
          if (l == 0) {
            const float hi = __uint_as_float((__float_as_uint(w) + 0x1000u) & 0xffffe000u);  // round to nearest TF32
            const int kt = tf32_row(k);
            reinterpret_cast<float*>(smem + a.img0_ofs[0])[((kt >> 2) * Np + n) * 4 + (kt & 3)] = hi;
            reinterpret_cast<__nv_bfloat16*>(smem + a.img1_ofs[0])[i8] = __float2bfloat16_rn(hi);
            reinterpret_cast<__nv_bfloat16*>(smem + a.img2_ofs[0])[i8] = __float2bfloat16_rn(w - hi);
          } else {
            const __half w1 = __float2half_rn(w);
            reinterpret_cast<__half*>(smem + a.img0_ofs[l])[i8] = w1;
            reinterpret_cast<__half*>(smem + a.img1_ofs[l])[i8] = __float2half_rn(w - __half2float(w1));
          }
        }
#pragma unroll
        for (int u = 0; u < RESTAGE_BATCH; ++u) v[u] = vn[u];
      }
      float* vec = reinterpret_cast<float*>(smem + a.vec_ofs);  // [0,64): scale, [64,128): 1/feat_thr
      if (tid < W) {
        vec[tid] = sc;
        vec[W + tid] = vt && a.feat_thr ? 1.0f / ft : 0.f;
      }
      if constexpr (X64) {  // zero past T: the zero-filled columns of an x tile stay exactly 0 through x * 0 + 0
        double* xab = reinterpret_cast<double*>(smem + a.xab_ofs);
        if (tid < W) {
          xab[tid] = vt ? __ldg(a.x_scale + (long)job.slot * TP + tid) : 0.0;
          xab[W + tid] = vt ? __ldg(a.x_offset + (long)job.slot * TP + tid) : 0.0;
        }
      }
      fence_proxy_async();  // generic-proxy writes above are read by the tensor cores (async proxy)
    }
    __syncthreads();

    // ---- the tiles of this item, warpgroup by warpgroup
    const float* vec = reinterpret_cast<const float*>(smem + a.vec_ofs);
    for (int tt = wg; tt < n_tiles; tt += NWG) {
      float d[32];
      uint32_t a1[4][4] = {}, a2[4][4] = {};
      // ---- layer 0
      {
        float xr[2][16];  // this thread's x: rows g, g+8 of its warp; per 16 columns the pairs 2t, 2t+1 and 2t+8, 2t+9
        mbar_wait(bar_x, x_phase);
        x_phase ^= 1;
        if constexpr (X64) {
          // x' = (float)(x * a + b): two roundings in double (no fma) and one to float, as gb_affine_f64 computes it.  Rows past the
          // end of x arrive as zeros and stay zeros, as in the float32 mode (columns past T do through a = b = 0).
          const double* xab = reinterpret_cast<const double*>(smem + a.xab_ofs);
          const long row0 = job.x_row + row_begin + tt * TILE + wq * 16 + g;
#pragma unroll
          for (int hr = 0; hr < 2; ++hr) {
            const bool live = row0 + 8 * hr < a.n_x_rows;
#pragma unroll
            for (int c = 0; c < 8; ++c) {
              const int col = 8 * c + 2 * t;
              const double2 v = *reinterpret_cast<const double2*>(xs + tile_ofs_x64(wq * 16 + g + 8 * hr, col));
              const double2 s = *reinterpret_cast<const double2*>(xab + col), o = *reinterpret_cast<const double2*>(xab + W + col);
              xr[hr][2 * c] = live ? (float)__dadd_rn(__dmul_rn(v.x, s.x), o.x) : 0.f;
              xr[hr][2 * c + 1] = live ? (float)__dadd_rn(__dmul_rn(v.y, s.y), o.y) : 0.f;
            }
          }
        } else {
#pragma unroll
          for (int hr = 0; hr < 2; ++hr)
#pragma unroll
            for (int c = 0; c < 8; ++c) {
              const float2 v = *reinterpret_cast<const float2*>(xs + tile_ofs(wq * 16 + g + 8 * hr, 8 * c + 2 * t));
              xr[hr][2 * c] = v.x;
              xr[hr][2 * c + 1] = v.y;
            }
        }
        // the y tile holds the staged outputs of the previous tile: every warp's stores must have read them before y is refilled
        if (lane == 0) bulk_wait_read<0>();
        warpgroup_sync(wg);  // the whole warpgroup has read x: the buffer takes the next tile's rows, which load behind this tile's layers
        if (leader) {
          if (tt + NWG < n_tiles) {
            if constexpr (X64) load_x64(tt + NWG);
            else load_tile(&a.tm_x, xbuf, bar_x, tt + NWG);
          }
          if (has_y) load_tile(&a.tm_y, ybuf, bar_y, tt);  // behind layers 1 ..
        }
        uint32_t xhi[4][8], alo[4][4], abf[4][4];
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {  // TF32 step 2 kk + hh: registers {row g, row g+8} x {col 2t, col 2t+1} of the pair 8 hh
            xhi[kk][4 * hh + 0] = __float_as_uint(trunc_tf32(xr[0][4 * kk + 2 * hh]));
            xhi[kk][4 * hh + 1] = __float_as_uint(trunc_tf32(xr[1][4 * kk + 2 * hh]));
            xhi[kk][4 * hh + 2] = __float_as_uint(trunc_tf32(xr[0][4 * kk + 2 * hh + 1]));
            xhi[kk][4 * hh + 3] = __float_as_uint(trunc_tf32(xr[1][4 * kk + 2 * hh + 1]));
          }
#pragma unroll
          for (int q = 0; q < 4; ++q) {  // 16-bit fragment: q = 0 (row g, cols 2t..), 1 (row g+8), 2 (row g, cols 2t+8..), 3 (row g+8, +8)
            const float v0 = xr[q & 1][4 * kk + 2 * (q >> 1)], v1 = xr[q & 1][4 * kk + 2 * (q >> 1) + 1];
            alo[kk][q] = pack_bf16(v0 - trunc_tf32(v0), v1 - trunc_tf32(v1));
            abf[kk][q] = pack_bf16(v0, v1);
          }
        }
        const int k16 = a.k16[0];
        const uint32_t i0 = sbase + a.img0_ofs[0], i1 = sbase + a.img1_ofs[0], i2 = sbase + a.img2_ofs[0];
        wgmma_fence();
        switch (a.Np[0]) {
          case 16: mma_layer0<16>(d, xhi, alo, abf, i0, i1, i2, k16); break;
          case 32: mma_layer0<32>(d, xhi, alo, abf, i0, i1, i2, k16); break;
          case 48: mma_layer0<48>(d, xhi, alo, abf, i0, i1, i2, k16); break;
          default: mma_layer0<64>(d, xhi, alo, abf, i0, i1, i2, k16); break;
        }
        wgmma_commit();
        wgmma_wait<0>();
        fence_acc(d);
        fence_frag(xhi);
        fence_frag(alo);
        fence_frag(abf);
      }

      // ---- hidden layers, then the output layer
      for (int l = 0; l < L; ++l) {
        if (l > 0) {
          const uint32_t i0 = sbase + a.img0_ofs[l], i1 = sbase + a.img1_ofs[l];
          const int k16 = a.k16[l];
          wgmma_fence();
          switch (a.Np[l]) {
            case 16: mma_hidden<16>(d, a1, a2, i0, i1, k16); break;
            case 32: mma_hidden<32>(d, a1, a2, i0, i1, k16); break;
            case 48: mma_hidden<48>(d, a1, a2, i0, i1, k16); break;
            default: mma_hidden<64>(d, a1, a2, i0, i1, k16); break;
          }
          wgmma_commit();
          wgmma_wait<0>();
          fence_acc(d);
          fence_frag(a1);
          fence_frag(a2);
        }
        if (l + 1 == L) break;
        // epilogue of hidden layer l: bias, tanh, FP16 pair -> A fragment of layer l + 1 (columns past N are 0: zero weights and bias)
        const float* bl = reinterpret_cast<const float*>(smem + a.bias_ofs[l]);
        const int nt = a.Np[l] >> 3;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          if (j < nt) {
            const float2 b = *reinterpret_cast<const float2*>(bl + 8 * j + 2 * t);
            const float v0 = tanh_from_scaled(fmaf(d[4 * j], TANH_ARG_SCALE, b.x)), v1 = tanh_from_scaled(fmaf(d[4 * j + 1], TANH_ARG_SCALE, b.y));
            const float v2 = tanh_from_scaled(fmaf(d[4 * j + 2], TANH_ARG_SCALE, b.x)), v3 = tanh_from_scaled(fmaf(d[4 * j + 3], TANH_ARG_SCALE, b.y));
            // n-tile j = columns 8j.. of the next layer's K: k-step j/2, fragment registers (j%2)*2 + {0: row g, 1: row g+8}
            split_f16(v0, v1, a1[j >> 1][2 * (j & 1)], a2[j >> 1][2 * (j & 1)]);
            split_f16(v2, v3, a1[j >> 1][2 * (j & 1) + 1], a2[j >> 1][2 * (j & 1) + 1]);
          }
        }
      }

      // ---- output layer: model output and every anomaly column, from the accumulator fragment
      const float* bo = reinterpret_cast<const float*>(smem + a.bias_ofs[L - 1]);
      const int wrow = row_begin + tt * TILE + wq * 16;  // row inside the job of the warp's first row
      const int trow = wrow + g;                         // ... and of fragment row g
      const int nt = a.Np[L - 1] >> 3;
      float2 yr[2][8];  // y in the accumulator's layout: rows g, g+8; columns 8j + 2t, + 1
      if (has_y) {
        mbar_wait(bar_y, y_phase);
        y_phase ^= 1;
#pragma unroll
        for (int hr = 0; hr < 2; ++hr)
#pragma unroll
          for (int j = 0; j < 8; ++j) yr[hr][j] = *reinterpret_cast<const float2*>(ys + tile_ofs(wq * 16 + g + 8 * hr, 8 * j + 2 * t));
      }
      // model output of fragment rows g + 8 hr, columns 8j + 2t, + 1 (the output layer's MMAs write no columns past Np).  The
      // accumulator registers are only read here: a write to them outside the MMAs makes ptxas serialise the wgmma chains.
      auto model_out = [&](int hr, int j) {
        const float2 b = *reinterpret_cast<const float2*>(bo + 8 * j + 2 * t);
        return j < nt ? make_float2(d[4 * j + 2 * hr] + b.x, d[4 * j + 2 * hr + 1] + b.y) : make_float2(0.f, 0.f);
      };

      // Per-tag outputs, one pass per array: model output, |y^ - y| (which then replaces y in registers), the same scaled, and
      // the same over the feature thresholds.  The passes over the unscaled and scaled arrays also sum the row totals, even when
      // the array itself is not asked for.  A pass stages its array's fragment in the warp's two 2 KB boxes, one per half of
      // 32 columns (with T <= 32 one box, the two boxes taking the arrays in turn), and lane 0 hands them to TMA stores.  A
      // store clips at the array's edges but not at the end of the job, whose next rows may belong to another job written by
      // another CTA: a warp whose 16 rows are not all inside the job copies its live rows out of the boxes itself.
      const int n_live = min(row_end - wrow, OBOX_ROWS);
      const bool want_su = has_y && a.o_totu, want_ss = has_y && (a.o_tots || a.o_totconf);
      float ss[2] = {0.f, 0.f}, su[2] = {0.f, 0.f};
      if (n_live > 0) {
        const int nh = TP > BOX_COLS ? 2 : 1;  // halves of 32 columns in a row
        int k = 0;                             // store groups issued in this tile
#pragma unroll
        for (int arr = 0; arr < 4; ++arr) {
          if (arr == 1 && has_y) {
#pragma unroll
            for (int hr = 0; hr < 2; ++hr)
#pragma unroll
              for (int j = 0; j < 8; ++j) {
                const float2 m = model_out(hr, j);
                yr[hr][j] = make_float2(fabsf(m.x - yr[hr][j].x), fabsf(m.y - yr[hr][j].y));
              }
          }
          float* o = arr == 0 ? a.o_model : arr == 1 ? a.o_tu : arr == 2 ? a.o_ts : a.o_conf;
          const bool put = o != nullptr && (arr == 0 || has_y);
          const bool acc = arr == 1 ? want_su : arr == 2 ? want_ss : false;
          if (!put && !acc) continue;
          const float* sv = vec + (arr == 3 ? W : 0);
          const uint32_t box0 = nh == 2 || (k & 1) == 0 ? obox0 : obox1;  // the box of columns 0..31; obox1 takes 32..63
          if (put) {
            if (lane == 0) {  // the stores that last used the box(es) have read them
              if (nh == 2 && k >= 1) bulk_wait_read<0>();
              if (nh == 1 && k >= 2) bulk_wait_read<1>();
            }
            __syncwarp();
          }
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            if (h == nh) break;
            uint8_t* bs = smem + ((h ? obox1 : box0) - sbase);
#pragma unroll
            for (int hr = 0; hr < 2; ++hr)
#pragma unroll
              for (int jj = 0; jj < 4; ++jj) {
                const int j = 4 * h + jj, col = 8 * j + 2 * t;
                float2 v = arr == 0 ? model_out(hr, j) : yr[hr][j];
                if (arr > 1) {
                  const float2 s = *reinterpret_cast<const float2*>(sv + col);
                  v = make_float2(v.x * s.x, v.y * s.y);
                }
                if (acc && col < TP) {  // T is a multiple of 4: col + 1 < T too
                  // rounding pinned to fma(x, x, y * y) and an add, so it does not depend on how the compiler contracts
                  const float q = __fmaf_rn(v.x, v.x, __fmul_rn(v.y, v.y));
                  if (arr == 1) su[hr] = __fadd_rn(su[hr], q);
                  else ss[hr] = __fadd_rn(ss[hr], q);
                }
                if (put) *reinterpret_cast<float2*>(bs + box_ofs(g + 8 * hr, 8 * jj + 2 * t)) = v;
              }
          }
          if (!put) continue;
          fence_proxy_async();  // the boxes are read by the TMA stores (async proxy)
          __syncwarp();
          if (n_live == OBOX_ROWS) {
            if (lane == 0) {
              for (int h = 0; h < nh; ++h) tma_store_2d(&a.tm_o[arr], h ? obox1 : box0, BOX_COLS * h, (int)(job.out_row + wrow));
              bulk_commit();
            }
          } else {
            for (int h = 0; h < nh; ++h) {
              const uint8_t* bs = smem + ((h ? obox1 : box0) - sbase);
              const int cols = min(BOX_COLS, TP - BOX_COLS * h);
              for (int i = lane; i < n_live * 8; i += 32) {  // 16-byte chunk c of row r: coalesced along the row
                const int r = i >> 3, c = i & 7;
                if (4 * c < cols)
                  __stcs(reinterpret_cast<float4*>(o + (job.out_row + wrow + r) * (long)TP + BOX_COLS * h + 4 * c),
                         *reinterpret_cast<const float4*>(bs + box_ofs(r, 4 * c)));
              }
            }
          }
          ++k;
        }
      }
      if (totals) {
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          ss[hr] += __shfl_xor_sync(0xffffffffu, ss[hr], 1);
          ss[hr] += __shfl_xor_sync(0xffffffffu, ss[hr], 2);
          su[hr] += __shfl_xor_sync(0xffffffffu, su[hr], 1);
          su[hr] += __shfl_xor_sync(0xffffffffu, su[hr], 2);
          const int r = trow + 8 * hr;
          if (t == 0 && r < row_end) {
            const long go = job.out_row + r;
            const float ts_ = ss[hr] * inv_w, tu_ = su[hr] * inv_w;
            if (a.o_tots) a.o_tots[go] = ts_;
            if (a.o_totu) a.o_totu[go] = tu_;
            if (a.o_totconf) a.o_totconf[go] = ts_ / __ldg(a.agg_thr + job.slot);
          }
        }
      }
    }
    __syncthreads();  // every warpgroup is done with this item's weights before the next item restages them
  }
  if (lane == 0) bulk_wait<0>();  // shared memory must outlive the stores' reads of it
}

// tile counters of the launches in flight: a ring of static device words, one per launch, zeroed stream-ordered before the kernel
// (no allocation; launches more than WORK_CTRS apart on the host never overlap on the device in practice)
constexpr int WORK_CTRS = 1024;
__device__ unsigned int g_work_ctr[WORK_CTRS];

// Shared-memory layout of the kernel for this architecture, x mode and warpgroup count (fills the shape and offset fields of
// `a`); returns its bytes.
int plan_smem(const gb_ffnet* net, TcArgs& a, bool x64 = false, int nwg = NWG_MAX) {
  const int L = net->n_layers;
  a.L = L;
  a.T = net->dims[0];
  int ofs = 0, pofs = 0;
  for (int l = 0; l < L; ++l) {
    a.K[l] = net->dims[l];
    a.N[l] = net->dims[l + 1];
    a.Np[l] = gb::round_up(a.N[l], 16);
    a.k16[l] = gb::round_up(a.K[l], 16) / 16;
    a.pofs[l] = pofs;
    pofs += a.K[l] * a.N[l] + a.N[l];
    const int kp = a.k16[l] * 16;
    a.img0_ofs[l] = ofs;  // layer 0: TF32 image [K/4][Np][4]; layers >= 1: FP16 w1 [K/8][Np][8]
    ofs += kp * a.Np[l] * (l == 0 ? 4 : 2);
    a.img1_ofs[l] = ofs;  // layer 0: BF16 of W_hi; layers >= 1: FP16 w2
    ofs += kp * a.Np[l] * 2;
    if (l == 0) {
      a.img2_ofs[l] = ofs;  // layer 0: BF16 of W - W_hi
      ofs += kp * a.Np[l] * 2;
    }
  }
  for (int l = 0; l < L; ++l) {
    a.bias_ofs[l] = ofs;
    ofs += W * 4;  // padded to the widest layer: the padded columns read zeros
  }
  a.w_bytes = gb::round_up(ofs, 16);
  ofs = a.w_bytes;
  a.vec_ofs = ofs; ofs += 2 * W * 4;
  if (x64) {
    a.xab_ofs = ofs; ofs += 2 * W * 8;
  }
  a.stage_ofs = ofs; ofs += 1024 + stage_bytes(x64, nwg);  // (the kernel aligns the tiles up to 1024 bytes inside this slack)
  return ofs;
}

constexpr int SMEM_MAX = 227 * 1024;

// Warpgroups of a launch with float64 x: three when their tiles fit next to this stack's weights (feedforward_hourglass(64) does
// not: 90 KB of weights), else two, whose tiles take the bytes of three float32 ones; 0 when neither fits.
int x64_warpgroups(const gb_ffnet* net, TcArgs& a, int* smem) {
  for (int nwg = NWG_MAX; nwg >= 2; --nwg) {
    *smem = plan_smem(net, a, true, nwg);
    if (*smem <= SMEM_MAX) return nwg;
  }
  return 0;
}

}  // namespace

extern "C" int gb_ffae_tc_supported(const gb_ffnet* net) {
  if (gb::validate_ffnet(net) != GB_OK) return GB_E_SHAPE;
  const int L = net->n_layers;
  if (L < 2 || L > MAXL || net->dims[0] != net->dims[L] || net->dims[0] > W || net->dims[0] < 24 || (net->dims[0] & 3)) {
    gb::set_error("tensor-core variant covers autoencoders of 24..%d tags (a multiple of 4) with at most %d layers", W, MAXL);
    return GB_E_SHAPE;
  }
  for (int l = 1; l < L; ++l)
    if (net->dims[l] > W) {
      gb::set_error("tensor-core variant needs hidden widths <= %d", W);
      return GB_E_SHAPE;
    }
  for (int l = 0; l < L; ++l)
    if (net->act[l] != (l + 1 < L ? GB_ACT_TANH : GB_ACT_LINEAR)) {
      gb::set_error("tensor-core variant is specialised for tanh hidden layers and a linear output (the factory defaults)");
      return GB_E_SHAPE;
    }
  TcArgs a{};
  const int smem = plan_smem(net, a);
  if (smem > SMEM_MAX) {
    gb::set_error("tensor-core variant: the weights and x / y tiles of this stack need %d bytes of shared memory (227 KB per SM)", smem);
    return GB_E_SHAPE;
  }
  return GB_OK;
}

// float64 x mode: the warpgroups its launch runs with (3 or 2), GB_E_SHAPE outside the variant's range, GB_E_SMEM when the
// stack's weights leave no room for two warpgroups' float64 x tiles.
extern "C" int gb_ffae_tc_warpgroups_x64(const gb_ffnet* net) {
  int rc = gb_ffae_tc_supported(net);
  if (rc != GB_OK) return rc;
  TcArgs a{};
  int smem = 0;
  const int nwg = x64_warpgroups(net, a, &smem);
  GB_REQUIRE(nwg > 0, GB_E_SMEM, "tensor-core variant with float64 x: the weights and two warpgroups' x / y tiles of this stack need %d "
             "bytes of shared memory (227 KB per SM)", smem);
  return nwg;
}

// x_scale == NULL: x is float32.  Otherwise x is float64 and x_scale / x_offset [n_slots][T] double are the slot's input scaler.
extern "C" int gb_ffae_infer_score_tc(const gb_ffnet* net, const float* params, const gb_job* jobs, int32_t n_jobs, int32_t max_rows,
                                      int64_t n_x_rows, int64_t n_out_rows, const void* x, const double* x_scale, const double* x_offset,
                                      const float* y, const float* scale, const float* feat_thr, const float* agg_thr, float* out_model,
                                      float* out_tag_scaled, float* out_tag_unscaled, float* out_total_scaled, float* out_total_unscaled,
                                      float* out_conf, float* out_total_conf, int32_t flags, void* stream) {
  int rc = gb_ffae_tc_supported(net);
  if (rc != GB_OK) return rc;
  GB_REQUIRE(flags == 0, GB_E_ARG, "variant bits above the low byte must be 0");
  GB_REQUIRE(n_x_rows > 0 && n_out_rows > 0, GB_E_ARG, "the tensor-core variant needs the row counts of x and of the outputs");
  const bool x64 = x_scale != nullptr;
  TcArgs a{};
  int nwg = NWG_MAX, smem_i = 0;
  if (x64) {
    nwg = gb_ffae_tc_warpgroups_x64(net);
    if (nwg < 0) return nwg;
    x64_warpgroups(net, a, &smem_i);
  } else {
    smem_i = plan_smem(net, a);
  }
  const size_t smem = (size_t)smem_i;
  GB_REQUIRE(n_x_rows < (1L << 31), GB_E_ARG, "%ld rows of x: TMA row coordinates are 32-bit", (long)n_x_rows);
  GB_REQUIRE(n_out_rows < (1L << 31), GB_E_ARG, "%ld output rows: TMA row coordinates are 32-bit", (long)n_out_rows);
  {
    CUresult r = x64 ? gb::sm90::encode_map_2d(&a.tm_x, CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 8, x, n_x_rows, a.T, BOX_COLS_X64, TILE)
                     : gb::sm90::encode_map_2d(&a.tm_x, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, x, n_x_rows, a.T, BOX_COLS, TILE);
    if (r == CUDA_SUCCESS && y) r = gb::sm90::encode_map_2d(&a.tm_y, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, y, n_x_rows, a.T, BOX_COLS, TILE);
    float* const outs[4] = {out_model, out_tag_unscaled, out_tag_scaled, out_conf};  // the order of TcArgs::tm_o
    for (int i = 0; i < 4; ++i)
      if (r == CUDA_SUCCESS && outs[i]) r = gb::sm90::encode_map_2d(&a.tm_o[i], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, outs[i], n_out_rows, a.T, BOX_COLS, OBOX_ROWS);
    GB_REQUIRE(r != CUDA_ERROR_NOT_FOUND, GB_E_CUDA, "cuTensorMapEncodeTiled is not available from the driver");
    GB_REQUIRE(r == CUDA_SUCCESS, GB_E_CUDA, "cuTensorMapEncodeTiled (x / y / outputs) failed with CUresult %d", (int)r);
  }

  int dev = 0, sms = 132;
  GB_CUDA_CHECK(cudaGetDevice(&dev));
  GB_CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const int tiles_per_job = (max_rows + TILE - 1) / TILE;
  a.tiles_per_job = tiles_per_job;
  a.n_jobs = n_jobs;
  a.pstride = (long)gb_ffnet_param_stride(net);
  a.params = params; a.jobs = jobs; a.y = y; a.scale = scale; a.feat_thr = feat_thr; a.agg_thr = agg_thr;
  a.o_model = out_model; a.o_ts = out_tag_scaled; a.o_tu = out_tag_unscaled; a.o_conf = out_conf;
  a.o_tots = out_total_scaled; a.o_totu = out_total_unscaled; a.o_totconf = out_total_conf;
  a.x_scale = x_scale; a.x_offset = x_offset; a.n_x_rows = (long)n_x_rows;

  const long g_total = (long)n_jobs * tiles_per_job;
  GB_REQUIRE(g_total < (1L << 31), GB_E_ARG, "%ld tiles in one launch: split the fleet", g_total);
  const int grid = (int)(g_total < sms ? g_total : sms);
  {
    static std::atomic<unsigned> next_ctr{0};
    void* base = nullptr;
    GB_CUDA_CHECK(cudaGetSymbolAddress(&base, g_work_ctr));
    a.work_ctr = static_cast<unsigned int*>(base) + (next_ctr.fetch_add(1) % WORK_CTRS);
    GB_CUDA_CHECK(cudaMemsetAsync(a.work_ctr, 0, sizeof(unsigned int), (cudaStream_t)stream));
  }
  auto launch = [&](auto kern, int nthreads) -> int {
    GB_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<grid, nthreads, smem, (cudaStream_t)stream>>>(a);
    return GB_OK;
  };
  rc = !x64 ? launch(ffae_tc_kernel<false, 3>, 384) : nwg == 3 ? launch(ffae_tc_kernel<true, 3>, 384) : launch(ffae_tc_kernel<true, 2>, 256);
  if (rc != GB_OK) return rc;
  GB_CUDA_CHECK(cudaGetLastError());
  return GB_OK;
}
