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

}  // namespace gb
