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
int validate_lstmnet(const gb_lstmnet* net);

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

// ---- optimizers (include/gordo_b200.h gb_optimizer; keras 3.3.3 keras/src/optimizers/*.py [3P], restated, not verified against TF)
// The fit kernels keep their own Adam for a NULL optimizer and for one that is plain Adam (no weight decay, no clipping), so
// those fits stay bit-identical; every other optimizer goes through opt_update.
inline int validate_optimizer(const gb_optimizer* o) {
  if (o == nullptr) return GB_OK;
  auto nonneg = [](float v) { return v >= 0.f && v < 3.0e38f; };  // false for NaN and inf
  auto unit = [](float v) { return v >= 0.f && v < 1.f; };
  GB_REQUIRE(o->kind >= GB_OPT_ADAM && o->kind <= GB_OPT_NADAM, GB_E_ARG, "optimizer kind=%d unknown (gb_opt: 0..6)", o->kind);
  GB_REQUIRE((o->flags & ~GB_OPT_CENTERED) == 0, GB_E_ARG, "optimizer flags=%d unknown", o->flags);
  GB_REQUIRE(!(o->flags & GB_OPT_CENTERED) || o->kind == GB_OPT_RMSPROP, GB_E_ARG, "optimizer flag GB_OPT_CENTERED is RMSprop's");
  GB_REQUIRE(!(o->flags & GB_OPT_CENTERED) || o->momentum == 0.f, GB_E_ARG,
             "optimizer: centered RMSprop with momentum needs a third state slot, which the fit kernels do not have");
  GB_REQUIRE(nonneg(o->lr) && nonneg(o->eps) && nonneg(o->momentum) && nonneg(o->initial_accumulator) && nonneg(o->weight_decay) &&
                 nonneg(o->clipvalue),
             GB_E_ARG, "optimizer lr/eps/momentum/initial_accumulator/weight_decay/clipvalue must be finite and >= 0");
  const bool two_betas = o->kind == GB_OPT_ADAM || o->kind == GB_OPT_ADAMW || o->kind == GB_OPT_ADAMAX || o->kind == GB_OPT_NADAM;
  GB_REQUIRE(o->kind == GB_OPT_ADAGRAD || unit(o->beta1), GB_E_ARG, "optimizer beta1/rho=%g outside [0, 1)", (double)o->beta1);
  GB_REQUIRE(!two_betas || unit(o->beta2), GB_E_ARG, "optimizer beta2=%g outside [0, 1)", (double)o->beta2);
  return GB_OK;
}
// Adam(W) without weight decay or clipping: the kernels' own Adam runs it, from the optimizer's lr / beta1 / beta2 / eps
inline bool plain_adam(const gb_optimizer* o) {
  return o == nullptr || ((o->kind == GB_OPT_ADAM || o->kind == GB_OPT_ADAMW) && o->weight_decay == 0.f && o->clipvalue == 0.f);
}

// Per-step scalars of optimizer step t, computed once per step off the per-parameter path.  nadam_p / nadam_pi carry Nadam's
// 0.96^t and the float32 product P_t, so that step t+1 follows from step t (opt_step_next) exactly as opt_step_at recomputes it
// from step 1: a fit split over several launches takes the same steps as one launch.
struct OptStep {
  float c0, c1, c2;  // ADAM(W): alpha_t = lr sqrt(1 - b2^t) / (1 - b1^t); ADAMAX: 1 / (1 - b1^t);
                     // NADAM: u_(t+1) / (1 - P_t u_(t+1)), (1 - u_t) / (1 - P_t), 1 / (1 - b2^t)
  int first;         // t == 1 (ADAGRAD reads initial_accumulator in place of its stored state)
  int t;
  float nadam_pi;
  double nadam_p;
};

__device__ __forceinline__ float nadam_u(float beta1, double p96) { return (float)((double)beta1 * (1.0 - 0.5 * p96)); }

__device__ __forceinline__ void opt_scalars(const gb_optimizer& o, OptStep& s) {
  const double t = (double)s.t;
  s.first = s.t == 1;
  switch (o.kind) {
    case GB_OPT_ADAMAX: s.c0 = (float)(1.0 / (1.0 - pow((double)o.beta1, t))); break;
    case GB_OPT_NADAM: {
      const float ut = nadam_u(o.beta1, s.nadam_p), ut1 = nadam_u(o.beta1, s.nadam_p * 0.96);
      s.c0 = ut1 / (1.f - s.nadam_pi * ut1);
      s.c1 = (1.f - ut) / (1.f - s.nadam_pi);
      s.c2 = (float)(1.0 / (1.0 - pow((double)o.beta2, t)));
      break;
    }
    default:
      s.c0 = (float)((double)o.lr * sqrt(1.0 - pow((double)o.beta2, t)) / (1.0 - pow((double)o.beta1, t)));
  }
}
// step prev.t + 1 from step prev.t
__device__ __forceinline__ OptStep opt_step_next(const gb_optimizer& o, const OptStep& prev) {
  OptStep s = prev;
  s.t = prev.t + 1;
  if (o.kind == GB_OPT_NADAM) {
    s.nadam_p = prev.nadam_p * 0.96;
    s.nadam_pi = prev.nadam_pi * nadam_u(o.beta1, s.nadam_p);
  }
  opt_scalars(o, s);
  return s;
}
// step t >= 1 from scratch: Nadam's product is taken from step 1, every other rule's scalars come from t alone
__device__ __forceinline__ OptStep opt_step_at(const gb_optimizer& o, int t) {
  OptStep s{};
  s.t = t - 1;
  s.nadam_pi = 1.f;  // P_0
  s.nadam_p = 1.0;   // 0.96^0
  if (o.kind == GB_OPT_NADAM)
    for (int k = 1; k < t; ++k) {
      s.nadam_p *= 0.96;
      s.nadam_pi *= nadam_u(o.beta1, s.nadam_p);
    }
  return opt_step_next(o, s);
}

// One parameter's update: w, its gradient g (summed over the mini-batch) and its two state slots.  Padded weight lanes (w = 0,
// g = 0) stay exactly zero under every rule.  The kind switch is uniform over a launch.
__device__ __forceinline__ void opt_update(const gb_optimizer& o, const OptStep& s, float& w, float g, float& s0, float& s1) {
  if (o.clipvalue > 0.f) g = fminf(fmaxf(g, -o.clipvalue), o.clipvalue);
  if (o.weight_decay != 0.f) w = __fsub_rn(w, __fmul_rn(__fmul_rn(w, o.weight_decay), o.lr));  // keras: w - w * wd * lr
  switch (o.kind) {
    case GB_OPT_RMSPROP: {
      s0 = o.beta1 * s0 + (1.f - o.beta1) * (g * g);
      float d;
      if (o.flags & GB_OPT_CENTERED) {
        s1 = o.beta1 * s1 + (1.f - o.beta1) * g;
        d = s0 - s1 * s1 + o.eps;
      } else {
        d = s0 + o.eps;
      }
      const float inc = o.lr * g / sqrtf(d);
      if (o.momentum > 0.f) {
        s1 = o.momentum * s1 + inc;
        w -= s1;
      } else {
        w -= inc;
      }
      break;
    }
    case GB_OPT_ADAGRAD: {
      s0 = (s.first ? o.initial_accumulator : s0) + g * g;
      w -= o.lr * g / sqrtf(s0 + o.eps);
      break;
    }
    case GB_OPT_ADADELTA: {
      s0 = o.beta1 * s0 + (1.f - o.beta1) * (g * g);
      const float dv = -(sqrtf(s1 + o.eps) * g / sqrtf(s0 + o.eps));
      s1 = o.beta1 * s1 + (1.f - o.beta1) * (dv * dv);
      w += o.lr * dv;
      break;
    }
    case GB_OPT_ADAMAX: {
      s0 += (g - s0) * (1.f - o.beta1);
      s1 = fmaxf(o.beta2 * s1, fabsf(g));
      w -= o.lr * s0 * s.c0 / (s1 + o.eps);
      break;
    }
    case GB_OPT_NADAM: {
      s0 += (g - s0) * (1.f - o.beta1);
      s1 += (g * g - s1) * (1.f - o.beta2);
      const float mhat = s.c0 * s0 + s.c1 * g;
      w -= mhat * o.lr / (sqrtf(s1 * s.c2) + o.eps);
      break;
    }
    default: {  // ADAM, ADAMW
      s0 += (g - s0) * (1.f - o.beta1);
      s1 += (g * g - s1) * (1.f - o.beta2);
      w -= s0 * s.c0 / (sqrtf(s1) + o.eps);
    }
  }
}

}  // namespace gb
