// Shared helpers for the gordo_b200 C-ABI library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string>
#include "../../include/gordo_b200.h"

namespace gb {

void set_error(const char* fmt, ...);

#define GB_CUDA_CHECK(expr)                                                              \
  do {                                                                                   \
    cudaError_t _e = (expr);                                                             \
    if (_e != cudaSuccess) {                                                             \
      gb::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return GB_E_CUDA;                                                                  \
    }                                                                                    \
  } while (0)

#define GB_REQUIRE(cond, code, ...)        \
  do {                                     \
    if (!(cond)) {                         \
      gb::set_error(__VA_ARGS__);          \
      return (code);                       \
    }                                      \
  } while (0)

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }
inline int round_up(int v, int m) { return (v + m - 1) / m * m; }

int validate_ffnet(const gb_ffnet* net);

// padded shared-memory image of one slot's Dense stack: W_l as [Kp][Np] (zero padded), then biases [Np]
struct FFImage {
  int kp[GB_MAX_LAYERS], np[GB_MAX_LAYERS];
  int wofs[GB_MAX_LAYERS], bofs[GB_MAX_LAYERS];  // offsets (floats) in the padded image
  int pofs[GB_MAX_LAYERS];                       // offset of W_l in the canonical parameter vector (bias follows)
  int total;                                     // floats in the padded image
  int max_np;                                    // widest padded activation
};
FFImage make_ff_image(const gb_ffnet* net, int pad);

__device__ __forceinline__ float apply_act(int act, float z) {
  switch (act) {
    case GB_ACT_TANH: return tanhf(z);
    case GB_ACT_RELU: return fmaxf(z, 0.f);
    case GB_ACT_SIGMOID: return 1.f / (1.f + expf(-z));
    default: return z;
  }
}
// derivative expressed through the layer output a = act(z)
__device__ __forceinline__ float act_grad_from_output(int act, float a) {
  switch (act) {
    case GB_ACT_TANH: return 1.f - a * a;
    case GB_ACT_RELU: return a > 0.f ? 1.f : 0.f;
    case GB_ACT_SIGMOID: return a * (1.f - a);
    default: return 1.f;
  }
}

// Keras regression losses other than mean squared error (keras 3.3.3 keras/src/losses/losses.py [3P], restated, not verified
// against TF): a per-element f of the prediction yh and the target t, averaged over the batch's elements by the caller, and
// its derivative with respect to yh.  e = yh - t, eps = 1e-7 (keras backend.epsilon()).  The fit kernels keep their own
// MSE arithmetic (d * d, 2 d / count) and call these for every other id.
constexpr float LOSS_EPS = 1e-7f;

__device__ __forceinline__ float softplus(float x) { return fmaxf(x, 0.f) + log1pf(expf(-fabsf(x))); }
__device__ __forceinline__ float sign0(float x) { return x > 0.f ? 1.f : (x < 0.f ? -1.f : 0.f); }  // TF's abs gradient: 0 at 0

__device__ __forceinline__ float loss_value(int loss, float yh, float t) {
  const float e = yh - t;
  switch (loss) {
    case GB_LOSS_MAE: return fabsf(e);
    case GB_LOSS_MAPE: return 100.f * fabsf(e) / fmaxf(fabsf(t), LOSS_EPS);
    case GB_LOSS_MSLE: {
      const float d = logf(fmaxf(yh, LOSS_EPS) + 1.f) - logf(fmaxf(t, LOSS_EPS) + 1.f);
      return d * d;
    }
    case GB_LOSS_HUBER: {  // delta = 1
      const float a = fabsf(e);
      return a <= 1.f ? 0.5f * e * e : a - 0.5f;
    }
    case GB_LOSS_LOG_COSH: return e + softplus(-2.f * e) - 0.69314718055994531f;
    default: return e * e;
  }
}

__device__ __forceinline__ float loss_grad(int loss, float yh, float t) {
  const float e = yh - t;
  switch (loss) {
    case GB_LOSS_MAE: return sign0(e);
    case GB_LOSS_MAPE: return 100.f * sign0(e) / fmaxf(fabsf(t), LOSS_EPS);
    case GB_LOSS_MSLE: {  // TF's maximum(yh, eps) passes the gradient to yh where yh >= eps
      if (!(yh >= LOSS_EPS)) return 0.f;
      const float p = yh + 1.f;
      return 2.f * (logf(p) - logf(fmaxf(t, LOSS_EPS) + 1.f)) / p;
    }
    case GB_LOSS_HUBER: return fabsf(e) <= 1.f ? e : sign0(e);
    case GB_LOSS_LOG_COSH: return 1.f - 2.f / (1.f + expf(2.f * e));  // 1 - 2 sigmoid(-2e)
    default: return 2.f * e;
  }
}

}  // namespace gb
