// The Dense fit kernels' shared definitions: the launch record FitArgs, the device helpers and the three kernel templates
// (ffae_fit_kernel, ffae_fit_reg_kernel, ffae_fit_drop_kernel) whose body is ffae_fit_body.cuh.  Included by ffae_fit.cu, which
// instantiates and launches the first two, and by ffae_fit_drop.cu, which holds the nine instantiations of the third in an object of
// their own (gb_fit::launch_drop), so that ffae_fit.o keeps exactly the kernels it had; ffae_fit_group.cu holds the grouped kernels
// of gb_ffae_fit_group, which take the same body and fill one record per group with ffae_fit.cu's setup_fit.
#pragma once
#include <cuda_pipeline.h>
#include <math_constants.h>
#include <type_traits>
#include "gb_common.cuh"

namespace gb_fit {

constexpr int THREADS = 512;
constexpr int NWARPS = THREADS / 32;
constexpr int BR = 32;  // rows of a mini-batch chunk: one row per lane

struct FitArgs {
  gb_ffnet net;
  gb::FFImage im;
  gb_fit_hparams hp;
  int apitch[GB_MAX_LAYERS + 1];  // pitch of activation buffer l (l = 0: x staging)
  int aofs[GB_MAX_LAYERS + 1];    // offset of activation buffer l (l >= 1) in smem floats
  int xofs[2], yofs[2], dofs[3];
  int gather_layer, gather_layer2;  // the two forward layers with the fewest tiles (the same layer twice in a one-layer stack): their idle warps issue the cp.async gather of the next chunk
  int d_global;  // how many of the three dz buffers (from the last one) live in the slot's L2-resident state area instead of shared memory
  int ypitch, dpitch;
  int wfloats, smem_floats;
  int n_in, n_out, max_rows;
  long pstride, sstride;
  float* params;
  float* adam_m;
  float* adam_v;
  const gb_job* jobs;
  const float *x, *y;
  const int32_t* perm;
  float *out_loss, *out_acc;
  long long* trace;  // debug (gb_debug_set_fit_trace): cycles of CTA 0 per phase, summed over the fit; NULL in production
  // gb_ffae_fit_split only (appended, so that the fields above keep their offsets in the parameter block of every kernel)
  const gb_fit_split* split;  // per job: held-out positions and row map; NULL = none
  const int32_t* row_map;
  int val_batch;
  float *out_val_loss, *out_val_acc;
  // gb_ffae_fit_stop only (appended too)
  const gb_fit_stop* stop;  // per job: the EarlyStopping rule; NULL = none
  float* best_params;       // [n_slots][pstride]: the snapshots
  int32_t *out_epochs, *out_best_epoch;
  // gb_ffae_fit_opt only (appended too): the optimizer of the OPT kernels
  gb_optimizer opt;
  // gb_ffae_fit_reg only (appended too): the weight regularizers of the REG kernels
  gb_dense_reg reg;
  // gb_ffae_fit_drop only (appended too): the dropout of the DROP kernels, per layer input l: bit l of drop_layers set when its rate
  // is not 0, the keep threshold floor(rate * 2^32) and the scale of the kept values (include/gordo_b200.h, gb_dense_dropout)
  uint32_t drop_layers;
  uint32_t drop_thr[GB_MAX_LAYERS];
  float drop_scale[GB_MAX_LAYERS];
};

enum FitEntry { FIT_PLAIN, FIT_SPLIT, FIT_STOP };

// the kernel family a fit runs: plain MSE with Adam, another loss, another optimizer than plain Adam, weight regularizers, dropout
enum FitFamily { FAMILY_MSE, FAMILY_LOSS, FAMILY_OPT, FAMILY_REG, FAMILY_DROP };

// ffae_fit_drop.cu: one launch of the ffae_fit_drop_kernel instantiation of (entry, memory plan), the plan as plan_fit chose it
int launch_drop(const FitArgs& a, FitEntry entry, bool w_global, size_t smem, int n_jobs, cudaStream_t stream);

// ffae_fit.cu, the host side of one net's fit, shared with gb_ffae_fit_group (ffae_fit_group.cu).  check_fit: the net, optimizer,
// pointer, hparams and alignment checks of launch_fit; check_split_stop / check_best_params: those of the split and stop entries;
// check_reg_drop: gb_ffae_fit_drop's checks of reg and drop against the net, and whether either record is more than zeros;
// fit_family: the family of the records that remain (NULL where they are zeros); setup_fit: the memory plan and the launch record.
int check_fit(const gb_ffnet* net, float* params, float* adam_m, float* adam_v, const gb_job* jobs, const float* x, const float* y,
              const int32_t* perm, const gb_fit_hparams* hp, float* out_loss, const gb_optimizer* opt);
int check_split_stop(const gb_fit_split* split, int32_t val_batch, const float* out_val_loss, const gb_fit_stop* stop,
                     const int32_t* out_epochs, const int32_t* out_best_epoch);
int check_best_params(const gb_fit_stop* stop, const float* best_params);
int check_reg_drop(const gb_ffnet* net, const gb_dense_reg* reg, const gb_dense_dropout* drop, bool& any_reg, bool& any_drop);
FitFamily fit_family(const gb_fit_hparams* hp, const gb_optimizer* opt, const gb_dense_reg* reg, const gb_dense_dropout* drop);
int setup_fit(const gb_ffnet* net, float* params, float* adam_m, float* adam_v, const gb_job* jobs, const gb_fit_split* split,
              int32_t max_rows, const float* x, const float* y, const int32_t* row_map, const int32_t* perm, const gb_fit_hparams* hp,
              int32_t val_batch, float* out_loss, float* out_acc, float* out_val_loss, float* out_val_acc, const gb_fit_stop* stop,
              float* best_params, int32_t* out_epochs, int32_t* out_best_epoch, const gb_optimizer* opt, const gb_dense_reg* reg,
              const gb_dense_dropout* drop, FitArgs& a, bool& w_global, size_t& smem);

}  // namespace gb_fit

namespace {

using gb_fit::BR;
using gb_fit::FitArgs;
using gb_fit::NWARPS;
using gb_fit::THREADS;

__device__ __forceinline__ uint32_t mix32(uint32_t h) {
  h ^= h >> 16; h *= 0x7feb352dU; h ^= h >> 15; h *= 0x846ca68bU; h ^= h >> 16;
  return h;
}

// dropout mask (include/gordo_b200.h, gb_dense_dropout): the word of row position p of the input of layer l under step key ks, and
// whether unit k of that row is kept
__device__ __forceinline__ uint32_t drop_row(uint32_t ks, int p, int l) {
  return mix32(ks + ((uint32_t)p * GB_MAX_LAYERS + (uint32_t)l) * 0x85ebca6bU);
}
__device__ __forceinline__ bool drop_keep(uint32_t kr, int k, uint32_t thr) { return mix32(kr + (uint32_t)k * 0x27d4eb2fU) >= thr; }

// keyed bijection on [0, n): 4-round Feistel network on the enclosing power of four, cycle-walked into range
__device__ __forceinline__ uint32_t permute_index(uint32_t i, uint32_t n, uint32_t key) {
  if (n <= 2) return (n == 2) ? (i ^ (key & 1u)) : 0u;
  int bits = 32 - __clz(n - 1);
  if (bits & 1) ++bits;
  const int half = bits >> 1;
  const uint32_t mask = (1u << half) - 1u;
  do {
    uint32_t l = i >> half, r = i & mask;
#pragma unroll
    for (int round = 0; round < 4; ++round) {
      const uint32_t t = l ^ (mix32(r * 0x9e3779b9U + key + round * 0x85ebca6bU) & mask);
      l = r;
      r = t;
    }
    i = (l << half) | r;
  } while (i >= n);
  return i;
}

// float -> unsigned with the same ordering (negative values below positive ones)
__device__ __forceinline__ unsigned order_key(float x) {
  const unsigned u = __float_as_uint(x);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ void adam_update(float& w, float g, float& m, float& v, float alpha, float omb1, float omb2,
                                            float eps) {
  m += (g - m) * omb1;
  v += (g * g - v) * omb2;
  float sq;
  asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(sq) : "f"(v));  // ~1 ulp, exact 0 at v = 0
  w -= __fdividef(alpha * m, sq + eps);
}

// acc[j][c]: partial sums of rows p + 8 j (j = 0..3) x 4 columns held by lane (p = lane & 7, kq = lane >> 3), to be summed over the four kq.
// Reduce-scatter in two rounds: the lanes 16 apart split rows {0,1} / {2,3}, then the lanes 8 apart split the remaining pair, so lane
// (p, kq) ends with the complete sums of row p + 8 kq (12 shuffles instead of 32 for an all-reduce).
__device__ __forceinline__ void quarter_reduce(const float (&acc)[4][4], int lane, float (&out)[4]) {
  const bool hi16 = (lane & 16) != 0, hi8 = (lane & 8) != 0;
  float h[2][4];
#pragma unroll
  for (int c = 0; c < 4; ++c) {
#pragma unroll
    for (int jj = 0; jj < 2; ++jj) {
      const float keep = hi16 ? acc[2 + jj][c] : acc[jj][c], send = hi16 ? acc[jj][c] : acc[2 + jj][c];
      h[jj][c] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
    }
  }
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const float keep = hi8 ? h[1][c] : h[0][c], send = hi8 ? h[0][c] : h[1][c];
    out[c] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
  }
}

// WG = false: the slot's padded weight image lives in shared memory for the whole fit (every 64-tag stack).  WG = true: the image does
// not fit beside the activations (e.g. the 128-tag hourglass, 245 KB) and lives in the slot's L2-resident state area instead; the
// code is the same, the loads become global.
// SPLIT (gb_ffae_fit_split): a job's rows are positions.  Training visits positions [0, n_rows); every epoch then ends with
// forward-only mini-batches of val_batch rows over the held-out positions [n_rows, n_rows + n_val), in order, whose loss and
// accuracy are the epoch's validation statistics.  Position p reads row x_row + row_map[map_ofs + p] (x_row + p without a map).
// The held-out batches are more chunks of the same visiting order, so the cp.async prefetch runs across them as well.
// STOP (gb_ffae_fit_stop, with SPLIT): Keras' EarlyStopping at the end of every epoch.  Thread 0 applies the job's rule to the
// monitored history entry it has just written and posts the decision (snapshot, stop) in s_red, free between two epoch_stats;
// one barrier shares it.  A snapshot is the weight image written to best_params in canonical layout; a job that stops drains
// its cp.async prefetch and leaves, so its SM takes the next job of the launch.
// LOSS (a fit whose hp.loss is not MSE): the output layer takes f / f' from gb::loss_value / gb::loss_grad.  Kept apart so that
// the MSE fits keep the exact code of the kernels without it.
// OPT (an optimizer other than plain Adam, gb_ffae_fit_opt; instantiated with LOSS only): the weight and bias updates are
// gb::opt_update on the two state slots (the Adam m / v loads and stores), with the per-step scalars gb::OptStep in place of
// the Adam step size, computed one step ahead as that is.
// REG (gb_ffae_fit_reg; instantiated with LOSS and OPT only, as ffae_fit_reg_kernel): Keras kernel / bias regularizers.  Their
// gradient joins the summed mini-batch gradient in the update loop, which also sums the penalty of the weights it writes, per thread and over real entries
// only: the next step's penalty is then ready without another pass (a pass over the canonical weights at the start of the launch
// seeds it).  Every thread adds rows * (its share of the penalty) to its acc_reg once per mini-batch, training or held-out, so the
// reduction of epoch_stats sums the penalty into the epoch's loss exactly as it sums the activity term.
// DROP (gb_ffae_fit_drop; instantiated with LOSS, OPT and REG only, as ffae_fit_drop_kernel): Keras Dropout on the inputs of the
// layers whose drop_layers bit is set, in training mini-batches only.  The staged x chunk is dropped in place before layer 0, a
// layer's activation as it is stored; input_grad regenerates the mask from the hash, zeroes the dropped elements' dz and takes a
// kept element's activation derivative at the stored value over the scale.  weight_step reads the stored (dropped) inputs as ever.
// The kernel body, shared by the three kernel templates below (every flag is a compile-time constant where it is included).  The
// REG and DROP kernels are templates of their own, so that the other kernels keep their six-flag names and their exact code.
// DG: some dz buffers live in global memory too (kept apart so that the usual case addresses them as shared memory)
template <bool WG, bool DG, bool SPLIT = false, bool STOP = false, bool LOSS = false, bool OPT = false>
__global__ void __launch_bounds__(THREADS, 1) ffae_fit_kernel(const FitArgs a) {
  constexpr bool REG = false, DROP = false;
#include "ffae_fit_body.cuh"
}

template <bool WG, bool DG, bool SPLIT, bool STOP>
__global__ void __launch_bounds__(THREADS, 1) ffae_fit_reg_kernel(const FitArgs a) {
  constexpr bool LOSS = true, OPT = true, REG = true, DROP = false;
#include "ffae_fit_body.cuh"
}

template <bool WG, bool DG, bool SPLIT, bool STOP>
__global__ void __launch_bounds__(THREADS, 1) ffae_fit_drop_kernel(const FitArgs a) {
  constexpr bool LOSS = true, OPT = true, REG = true, DROP = true;
#include "ffae_fit_body.cuh"
}

}  // namespace
