// Library-level entry points + dispatch of gb_ffae_infer_score between kernel variants.
#include <stdarg.h>
#include "gb_common.cuh"

namespace gb {

static thread_local std::string g_last_error;

void set_error(const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_last_error = buf;
}

int validate_ffnet(const gb_ffnet* net) {
  GB_REQUIRE(net != nullptr, GB_E_ARG, "net is NULL");
  GB_REQUIRE(net->n_layers >= 1 && net->n_layers <= GB_MAX_LAYERS, GB_E_SHAPE, "n_layers=%d outside [1,%d]",
             net->n_layers, GB_MAX_LAYERS);
  for (int l = 0; l <= net->n_layers; ++l)
    GB_REQUIRE(net->dims[l] >= 1 && net->dims[l] <= GB_MAX_WIDTH, GB_E_SHAPE, "dims[%d]=%d outside [1,%d]", l,
               net->dims[l], GB_MAX_WIDTH);
  for (int l = 0; l < net->n_layers; ++l)
    GB_REQUIRE(net->act[l] >= GB_ACT_LINEAR && net->act[l] <= GB_ACT_SIGMOID, GB_E_ARG, "act[%d]=%d unknown", l,
               net->act[l]);
  return GB_OK;
}

// the LSTM stacks every inference and fit kernel takes
constexpr int LSTM_MAX_UNITS = 512;
constexpr int LSTM_MAX_FEATURES = 512;

int validate_lstmnet(const gb_lstmnet* net) {
  GB_REQUIRE(net != nullptr, GB_E_ARG, "net is NULL");
  GB_REQUIRE(net->n_layers >= 1 && net->n_layers <= GB_MAX_LAYERS, GB_E_SHAPE, "n_layers=%d outside [1,%d]",
             net->n_layers, GB_MAX_LAYERS);
  GB_REQUIRE(net->n_features >= 1 && net->n_features <= LSTM_MAX_FEATURES && net->n_features_out >= 1 &&
                 net->n_features_out <= LSTM_MAX_FEATURES,
             GB_E_SHAPE, "n_features/n_features_out outside [1,%d]", LSTM_MAX_FEATURES);
  GB_REQUIRE(net->lookback >= 1, GB_E_ARG, "lookback=%d must be >= 1", net->lookback);
  for (int l = 0; l < net->n_layers; ++l) {
    GB_REQUIRE(net->units[l] >= 1 && net->units[l] <= LSTM_MAX_UNITS, GB_E_SHAPE, "units[%d]=%d outside [1,%d]", l,
               net->units[l], LSTM_MAX_UNITS);
    GB_REQUIRE(net->act[l] >= GB_ACT_LINEAR && net->act[l] <= GB_ACT_SIGMOID, GB_E_ARG, "act[%d] unknown", l);
  }
  return GB_OK;
}

FFImage make_ff_image(const gb_ffnet* net, int pad) {
  FFImage im{};
  int ofs = 0, pofs = 0, max_np = round_up(net->dims[0], pad);
  for (int l = 0; l < net->n_layers; ++l) {
    im.kp[l] = round_up(net->dims[l], pad);
    im.np[l] = round_up(net->dims[l + 1], pad);
    im.wofs[l] = ofs;
    ofs += im.kp[l] * im.np[l];
    im.bofs[l] = ofs;
    ofs += im.np[l];
    im.pofs[l] = pofs;
    pofs += net->dims[l] * net->dims[l + 1] + net->dims[l + 1];
    if (im.np[l] > max_np) max_np = im.np[l];
  }
  im.total = ofs;
  im.max_np = max_np;
  return im;
}

}  // namespace gb

extern "C" {

int gb_abi_version(void) { return GB_ABI_VERSION; }

const char* gb_last_error(void) { return gb::g_last_error.c_str(); }

int gb_device_check(int device, int* sm_count) {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0) {
    gb::set_error("no CUDA device: %s", cudaGetErrorString(e));
    return GB_E_DEVICE;
  }
  GB_REQUIRE(device >= 0 && device < n, GB_E_ARG, "device %d out of range (%d devices)", device, n);
  cudaDeviceProp p;
  GB_CUDA_CHECK(cudaGetDeviceProperties(&p, device));
  if (sm_count) *sm_count = p.multiProcessorCount;
  GB_REQUIRE(p.major == 9 && p.minor == 0, GB_E_DEVICE, "device %d is sm_%d%d; this library is built for sm_90a (H100) only", device,
             p.major, p.minor);
  return GB_OK;
}

size_t gb_ffnet_param_count(const gb_ffnet* net) {
  if (gb::validate_ffnet(net) != GB_OK) return 0;
  size_t n = 0;
  for (int l = 0; l < net->n_layers; ++l) n += (size_t)net->dims[l] * net->dims[l + 1] + net->dims[l + 1];
  return n;
}

size_t gb_ffnet_param_stride(const gb_ffnet* net) { return (gb_ffnet_param_count(net) + 3) / 4 * 4; }

// kernel variants (defined in their own translation units); x_scale == NULL: x is float32, else float64 through the input scaler
int gb_ffae_infer_score_fma(const gb_ffnet*, const float*, const gb_job*, int32_t, int32_t, const void*, const double*, const double*,
                            const float*, const float*, const float*, const float*, float*, float*, float*, float*, float*, float*,
                            float*, void*);
int gb_ffae_small_supported(const gb_ffnet*);
int gb_ffae_infer_score_small(const gb_ffnet*, const float*, const gb_job*, int32_t, int32_t, const void*, const double*, const double*,
                              const float*, const float*, const float*, const float*, float*, float*, float*, float*, float*, float*,
                              float*, void*);
int gb_ffae_infer_score_tc(const gb_ffnet*, const float*, const gb_job*, int32_t, int32_t, int64_t, int64_t, const void*, const double*,
                           const double*, const float*, const float*, const float*, const float*, float*, float*, float*, float*, float*,
                           float*, float*, int32_t, void*);
int gb_ffae_tc_warpgroups_x64(const gb_ffnet*);

}  // extern "C"

namespace {

int infer_score(const gb_ffnet* net, const float* params, const gb_job* jobs, int32_t n_jobs, int32_t max_rows, int64_t n_x_rows,
                int64_t n_out_rows, const void* x, const double* x_scale, const double* x_offset, const float* y, const float* scale,
                const float* feat_thr, const float* agg_thr, float* out_model, float* out_tag_scaled, float* out_tag_unscaled,
                float* out_total_scaled, float* out_total_unscaled, float* out_conf, float* out_total_conf, int32_t variant,
                void* stream) {
  int rc = gb::validate_ffnet(net);
  if (rc != GB_OK) return rc;
  GB_REQUIRE(params && jobs && x && out_model, GB_E_ARG, "params/jobs/x/out_model must be non-NULL");
  GB_REQUIRE(n_jobs >= 0 && max_rows >= 0, GB_E_ARG, "negative n_jobs/max_rows");
  const int32_t tc_flags = variant >> 8;
  variant &= 0xff;
  GB_REQUIRE(variant >= 0 && variant <= 3, GB_E_ARG, "variant=%d unknown", variant);
  if (y == nullptr)
    GB_REQUIRE(!out_tag_scaled && !out_tag_unscaled && !out_total_scaled && !out_total_unscaled && !out_conf &&
                   !out_total_conf,
               GB_E_ARG, "score outputs requested without y");
  else
    GB_REQUIRE(scale != nullptr || (!out_tag_scaled && !out_total_scaled && !out_total_conf), GB_E_ARG,
               "scaled outputs requested without scale");
  GB_REQUIRE(!out_conf || feat_thr, GB_E_ARG, "out_conf requested without feat_thr");
  GB_REQUIRE(!out_total_conf || (agg_thr && scale), GB_E_ARG, "out_total_conf requested without agg_thr/scale");
  const void* ptrs[] = {params, x, y, out_model, out_tag_scaled, out_tag_unscaled, out_conf};
  for (const void* p : ptrs) GB_REQUIRE(gb::aligned16(p), GB_E_ALIGN, "array pointer %p is not 16-byte aligned", p);
  if (n_jobs == 0 || max_rows == 0) return GB_OK;
  bool tc_ok = gb_ffae_tc_supported(net) == GB_OK;
  if (variant == 2 && !tc_ok) return GB_E_SHAPE;
  if (variant == 2 || (variant == 0 && tc_ok))
    return gb_ffae_infer_score_tc(net, params, jobs, n_jobs, max_rows, n_x_rows, n_out_rows, x, x_scale, x_offset, y, scale, feat_thr,
                                  agg_thr, out_model, out_tag_scaled, out_tag_unscaled, out_total_scaled, out_total_unscaled, out_conf,
                                  out_total_conf, tc_flags, stream);
  const bool small_ok = gb_ffae_small_supported(net) == GB_OK;
  if (variant == 3 && !small_ok) return GB_E_SHAPE;
  if (variant == 3 || (variant == 0 && small_ok))
    return gb_ffae_infer_score_small(net, params, jobs, n_jobs, max_rows, x, x_scale, x_offset, y, scale, feat_thr, agg_thr, out_model,
                                     out_tag_scaled, out_tag_unscaled, out_total_scaled, out_total_unscaled, out_conf, out_total_conf,
                                     stream);
  return gb_ffae_infer_score_fma(net, params, jobs, n_jobs, max_rows, x, x_scale, x_offset, y, scale, feat_thr, agg_thr, out_model,
                                 out_tag_scaled, out_tag_unscaled, out_total_scaled, out_total_unscaled, out_conf, out_total_conf,
                                 stream);
}

}  // namespace

extern "C" {

int gb_ffae_infer_score(const gb_ffnet* net, const float* params, const gb_job* jobs, int32_t n_jobs, int32_t max_rows,
                        int64_t n_x_rows, int64_t n_out_rows, const float* x, const float* y, const float* scale, const float* feat_thr,
                        const float* agg_thr, float* out_model, float* out_tag_scaled, float* out_tag_unscaled,
                        float* out_total_scaled, float* out_total_unscaled, float* out_conf, float* out_total_conf,
                        int32_t variant, void* stream) {
  return infer_score(net, params, jobs, n_jobs, max_rows, n_x_rows, n_out_rows, x, nullptr, nullptr, y, scale, feat_thr, agg_thr,
                     out_model, out_tag_scaled, out_tag_unscaled, out_total_scaled, out_total_unscaled, out_conf, out_total_conf, variant,
                     stream);
}

int gb_ffae_infer_score_x64(const gb_ffnet* net, const float* params, const gb_job* jobs, int32_t n_jobs, int32_t max_rows,
                            int64_t n_x_rows, int64_t n_out_rows, const double* x, const double* x_scale, const double* x_offset,
                            const float* y, const float* scale, const float* feat_thr, const float* agg_thr, float* out_model,
                            float* out_tag_scaled, float* out_tag_unscaled, float* out_total_scaled, float* out_total_unscaled,
                            float* out_conf, float* out_total_conf, int32_t variant, void* stream) {
  GB_REQUIRE(x_scale && x_offset, GB_E_ARG, "x_scale/x_offset must be non-NULL");
  return infer_score(net, params, jobs, n_jobs, max_rows, n_x_rows, n_out_rows, x, x_scale, x_offset, y, scale, feat_thr, agg_thr,
                     out_model, out_tag_scaled, out_tag_unscaled, out_total_scaled, out_total_unscaled, out_conf, out_total_conf, variant,
                     stream);
}

int gb_ffae_infer_plan_x64(const gb_ffnet* net, int32_t variant, int32_t* kernel, int32_t* tc_warpgroups) {
  int rc = gb::validate_ffnet(net);
  if (rc != GB_OK) return rc;
  GB_REQUIRE(variant >= 0 && variant <= 3, GB_E_ARG, "variant=%d unknown (debug bits above the low byte are not part of a plan)", variant);
  int k = variant, nwg = 0;
  if (k == 0) k = gb_ffae_tc_supported(net) == GB_OK ? 2 : gb_ffae_small_supported(net) == GB_OK ? 3 : 1;
  if (k == 2) {
    nwg = gb_ffae_tc_warpgroups_x64(net);
    if (nwg < 0) return nwg;
  } else if (k == 3) {
    if (gb_ffae_small_supported(net) != GB_OK) return GB_E_SHAPE;
  } else {
    rc = gb_ffae_infer_plan(net, nullptr, nullptr);
    if (rc != GB_OK) return rc;
  }
  if (kernel) *kernel = k;
  if (tc_warpgroups) *tc_warpgroups = nwg;
  return GB_OK;
}

}  // extern "C"
