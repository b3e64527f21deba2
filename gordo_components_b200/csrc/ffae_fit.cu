// K2: fit of the Dense autoencoder stacks -- one persistent CTA per job trains the whole fit.
//
// Replaces scikeras KerasRegressor.fit -> keras Model.fit (gordo/machine/model/models.py:284) for
// the networks of factories/feedforward_autoencoder.py:65-104:
//   loss = mean(f(net(x), y)) + sum_l l1[l]*sum|a_l|,  Adam(lr, b1, b2, eps) [keras defaults 1e-3/.9/.999/1e-7],
//   f = (net(x)-y)^2 or another Keras regression loss (hp.loss, gb::loss_value / gb::loss_grad),
//   every epoch visits a permutation of the job's rows in batches of batch_size (last partial batch kept).
//
// A fit is a chain of epochs*ceil(n/batch) dependent optimizer steps of ~3 MFLOP each, so it is latency bound,
// not roofline bound: the design keeps everything a step needs on chip.  The slot's weights live in shared
// memory (padded [Kp][Np] image) for the entire fit, every layer's activations of the current mini-batch stay in
// shared memory for the backward pass, the next mini-batch is gathered with cp.async while the current one is
// processed, and the Adam moments (opaque state, same padded layout) stream through L2.  Machines (and CV folds,
// which are just more jobs) are independent, so the grid is simply one CTA per job.
// A mini-batch larger than 32 rows is processed as chunks of 32: the chunks' weight gradients are summed in
// an L2-resident scratch image (second half of the opaque Adam-m state) and the optimizer runs with the last chunk.
// The two products with the batch rows as the outer dimension (a.W and dz.W^T) give a lane four rows and a quarter of the reduction
// index (4x4 register tile, reduce-scatter over the four quarters); the weight gradient gives a thread a 4x2 block of W.
#include "ffae_fit_kernels.cuh"

namespace {

using gb_fit::FIT_PLAIN;
using gb_fit::FIT_SPLIT;
using gb_fit::FIT_STOP;
using gb_fit::FitEntry;

// the kernel of one dispatch cell: REG takes the regularized kernels (LOSS and OPT implied); the dropout kernels are launched by
// gb_fit::launch_drop (ffae_fit_drop.cu)
template <bool WG, bool DG, bool SPLIT, bool STOP, bool LOSS, bool OPT, bool REG>
constexpr auto fit_kernel() {
  if constexpr (REG) return &ffae_fit_reg_kernel<WG, DG, SPLIT, STOP>;
  else return &ffae_fit_kernel<WG, DG, SPLIT, STOP, LOSS, OPT>;
}

long long* g_fit_trace = nullptr;

int odd_pitch(int width) {
  int p4 = (width + 3) / 4;
  if ((p4 & 1) == 0) ++p4;
  return p4 * 4;
}

// A block may opt into 227 KB of shared memory, static and dynamic together: cudaFuncSetAttribute refuses a dynamic size that
// leaves less than the kernel's static arrays (s_red, s_alpha, s_opt, s_idx, s_phase of ffae_fit_body.cuh: 752 bytes, 808 with
// OPT; cuobjdump -res-usage reports 1776 / 1824, adding the 1 KB sm_90 reserves for every block).  The plans keep 2 KB for them,
// which covers either count; tests/test_fit_widths_host.py checks the reported sizes against it.
constexpr size_t FIT_STATIC_SMEM = 2048;
constexpr size_t FIT_DYNAMIC_SMEM = 227 * 1024 - FIT_STATIC_SMEM;

// Memory plan of a fit: the first of five layouts that fits.  Everything in shared memory; else the weight image in the slot's
// L2-resident state area; then, one by one, the dz buffers in L2 as well (at most as many as the two spare thirds of the Adam-v
// area hold).  Fills the layout fields of `a` (net, image, widths, offsets, pitches, d_global) and the dynamic shared memory.
int plan_fit(const gb_ffnet* net, FitArgs& a, bool& w_global, size_t& smem) {
  a.net = *net;
  a.im = gb::make_ff_image(net, 4);
  const int L = net->n_layers;
  a.n_in = net->dims[0];
  a.n_out = net->dims[L];
  a.wfloats = gb::round_up(a.im.total, 4);
  smem = 0;
  w_global = false;
  for (int pass = 0; pass < 5; ++pass) {
    w_global = pass >= 1;
    a.d_global = pass >= 2 ? pass - 1 : 0;
    int ofs = w_global ? 0 : a.wfloats;
    a.apitch[0] = odd_pitch(a.im.kp[0]);
    for (int l = 1; l <= L; ++l) {
      a.apitch[l] = odd_pitch(a.im.np[l - 1]);
      a.aofs[l] = ofs;
      ofs += BR * a.apitch[l];
    }
    for (int b = 0; b < 2; ++b) { a.xofs[b] = ofs; ofs += BR * a.apitch[0]; }
    a.ypitch = odd_pitch(gb::round_up(a.n_out, 4));
    for (int b = 0; b < 2; ++b) { a.yofs[b] = ofs; ofs += BR * a.ypitch; }
    a.dpitch = odd_pitch(a.im.max_np);
    for (int b = 0; b < 3 - a.d_global; ++b) { a.dofs[b] = ofs; ofs += BR * a.dpitch; }
    a.smem_floats = ofs;
    smem = (size_t)ofs * sizeof(float);
    if (smem <= FIT_DYNAMIC_SMEM && (long)a.d_global * BR * a.dpitch <= 2L * a.wfloats) break;
  }
  GB_REQUIRE(smem <= FIT_DYNAMIC_SMEM && (long)a.d_global * BR * a.dpitch <= 2L * a.wfloats, GB_E_SMEM,
             "architecture needs %zu bytes of shared memory for the activations of one mini-batch chunk (at most %zu)", smem,
             FIT_DYNAMIC_SMEM);
  return GB_OK;
}


// gb_ffae_fit (FIT_PLAIN: the kernels without the held-out pass), gb_ffae_fit_split and gb_ffae_fit_stop
int launch_fit(const gb_ffnet* net, float* params, float* adam_m, float* adam_v, const gb_job* jobs, const gb_fit_split* split,
               int32_t n_jobs, int32_t max_rows, const float* x, const float* y, const int32_t* row_map, const int32_t* perm,
               const gb_fit_hparams* hp, int32_t val_batch, float* out_loss, float* out_acc, float* out_val_loss, float* out_val_acc,
               const gb_fit_stop* stop, float* best_params, int32_t* out_epochs, int32_t* out_best_epoch, FitEntry entry,
               const gb_optimizer* opt, const gb_dense_reg* reg, const gb_dense_dropout* drop, void* stream) {
  int rc = gb_fit::check_fit(net, params, adam_m, adam_v, jobs, x, y, perm, hp, out_loss, opt);
  if (rc != GB_OK) return rc;
  if (n_jobs == 0 || max_rows == 0) return GB_OK;

  FitArgs a{};
  size_t smem = 0;
  bool w_global = false;
  rc = gb_fit::setup_fit(net, params, adam_m, adam_v, jobs, split, max_rows, x, y, row_map, perm, hp, val_batch, out_loss, out_acc,
                         out_val_loss, out_val_acc, stop, best_params, out_epochs, out_best_epoch, opt, reg, drop, a, w_global, smem);
  if (rc != GB_OK) return rc;
  a.trace = g_fit_trace;
  auto launch = [&](auto kernel) -> int {
    GB_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kernel<<<n_jobs, THREADS, smem, (cudaStream_t)stream>>>(a);
    return GB_OK;
  };
  auto dispatch = [&](auto any_loss, auto any_opt, auto any_reg) -> int {
    constexpr bool LS = decltype(any_loss)::value, OP = decltype(any_opt)::value, RG = decltype(any_reg)::value;
    if (entry == FIT_STOP) {
      if (a.d_global > 0) return launch(fit_kernel<true, true, true, true, LS, OP, RG>());
      if (w_global) return launch(fit_kernel<true, false, true, true, LS, OP, RG>());
      return launch(fit_kernel<false, false, true, true, LS, OP, RG>());
    }
    if (entry == FIT_SPLIT) {
      if (a.d_global > 0) return launch(fit_kernel<true, true, true, false, LS, OP, RG>());
      if (w_global) return launch(fit_kernel<true, false, true, false, LS, OP, RG>());
      return launch(fit_kernel<false, false, true, false, LS, OP, RG>());
    }
    if (a.d_global > 0) return launch(fit_kernel<true, true, false, false, LS, OP, RG>());
    if (w_global) return launch(fit_kernel<true, false, false, false, LS, OP, RG>());
    return launch(fit_kernel<false, false, false, false, LS, OP, RG>());
  };
  // another optimizer than plain Adam takes the LOSS kernels (their loss switch covers MSE), so it adds 9 instantiations, not 18;
  // weight regularizers take the 9 ffae_fit_reg_kernel instantiations, dropout the 9 ffae_fit_drop_kernel ones (ffae_fit_drop.cu)
  const std::false_type no{};
  const std::true_type yes{};
  switch (gb_fit::fit_family(hp, opt, reg, drop)) {
    case gb_fit::FAMILY_DROP: rc = gb_fit::launch_drop(a, entry, w_global, smem, n_jobs, (cudaStream_t)stream); break;
    case gb_fit::FAMILY_REG: rc = dispatch(yes, yes, yes); break;
    case gb_fit::FAMILY_OPT: rc = dispatch(yes, yes, no); break;
    case gb_fit::FAMILY_MSE: rc = dispatch(no, no, no); break;
    default: rc = dispatch(yes, no, no);
  }
  if (rc != GB_OK) return rc;
  GB_CUDA_CHECK(cudaGetLastError());
  return GB_OK;
}

}  // namespace

extern "C" {

size_t gb_ffae_fit_state_stride(const gb_ffnet* net) {
  if (gb::validate_ffnet(net) != GB_OK) return 0;
  return 3 * (size_t)gb::round_up(gb::make_ff_image(net, 4).total, 4);  // moments + gradient scratch of multi-chunk mini-batches + weight image of wide stacks
}

int gb_ffae_fit_plan(const gb_ffnet* net, int32_t* weights_in_l2, int32_t* dz_in_l2) {
  const int rc = gb::validate_ffnet(net);
  if (rc != GB_OK) return rc;
  FitArgs a{};
  size_t smem = 0;
  bool w_global = false;
  if (plan_fit(net, a, w_global, smem) != GB_OK) return GB_E_SMEM;
  if (weights_in_l2) *weights_in_l2 = w_global ? 1 : 0;
  if (dz_in_l2) *dz_in_l2 = a.d_global;
  return GB_OK;
}

// debug aid (not part of the public header): per-phase cycle sums of CTA 0 into a device buffer of 2*GB_MAX_LAYERS+4 int64
// (0 gather wait, 1..L forward layers, L+1 loss, L+2.. backward phases, 2L+2 set-up, 2L+3 tail); NULL switches it off
int gb_debug_set_fit_trace(void* dev_buf) {
  g_fit_trace = static_cast<long long*>(dev_buf);
  return GB_OK;
}

int gb_ffae_fit(const gb_ffnet* net, float* params, float* adam_m, float* adam_v, const gb_job* jobs, int32_t n_jobs,
                int32_t max_rows, const float* x, const float* y, const int32_t* perm, const gb_fit_hparams* hp,
                float* out_loss, float* out_acc, void* stream) {
  return launch_fit(net, params, adam_m, adam_v, jobs, nullptr, n_jobs, max_rows, x, y, nullptr, perm, hp, 1, out_loss, out_acc,
                    nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, FIT_PLAIN, nullptr, nullptr, nullptr, stream);
}

int gb_ffae_fit_split(const gb_ffnet* net, float* params, float* adam_m, float* adam_v, const gb_job* jobs,
                      const gb_fit_split* split, int32_t n_jobs, int32_t max_rows, const float* x, const float* y,
                      const int32_t* row_map, const int32_t* perm, const gb_fit_hparams* hp, int32_t val_batch,
                      float* out_loss, float* out_acc, float* out_val_loss, float* out_val_acc, void* stream) {
  GB_REQUIRE(!split || out_val_loss, GB_E_ARG, "split needs out_val_loss");
  GB_REQUIRE(!split || val_batch >= 1, GB_E_ARG, "val_batch=%d must be >= 1", val_batch);
  return launch_fit(net, params, adam_m, adam_v, jobs, split, n_jobs, max_rows, x, y, row_map, perm, hp, split ? val_batch : 1,
                    out_loss, out_acc, out_val_loss, out_val_acc, nullptr, nullptr, nullptr, nullptr, FIT_SPLIT, nullptr, nullptr, nullptr, stream);
}

int gb_ffae_fit_stop(const gb_ffnet* net, float* params, float* adam_m, float* adam_v, const gb_job* jobs,
                     const gb_fit_split* split, int32_t n_jobs, int32_t max_rows, const float* x, const float* y,
                     const int32_t* row_map, const int32_t* perm, const gb_fit_hparams* hp, int32_t val_batch,
                     float* out_loss, float* out_acc, float* out_val_loss, float* out_val_acc, const gb_fit_stop* stop,
                     float* best_params, int32_t* out_epochs, int32_t* out_best_epoch, void* stream) {
  GB_REQUIRE(!split || out_val_loss, GB_E_ARG, "split needs out_val_loss");
  GB_REQUIRE(!split || val_batch >= 1, GB_E_ARG, "val_batch=%d must be >= 1", val_batch);
  GB_REQUIRE(!stop || (best_params && out_epochs && out_best_epoch), GB_E_ARG,
             "stop needs best_params, out_epochs and out_best_epoch");
  GB_REQUIRE(!stop || gb::aligned16(best_params), GB_E_ARG, "best_params must be 16-byte aligned");
  return launch_fit(net, params, adam_m, adam_v, jobs, split, n_jobs, max_rows, x, y, row_map, perm, hp, split ? val_batch : 1,
                    out_loss, out_acc, out_val_loss, out_val_acc, stop, best_params, out_epochs, out_best_epoch, FIT_STOP, nullptr, nullptr, nullptr, stream);
}

int gb_ffae_fit_drop(const gb_ffnet* net, float* params, float* adam_m, float* adam_v, const gb_job* jobs,
                     const gb_fit_split* split, int32_t n_jobs, int32_t max_rows, const float* x, const float* y,
                     const int32_t* row_map, const int32_t* perm, const gb_fit_hparams* hp, int32_t val_batch,
                     float* out_loss, float* out_acc, float* out_val_loss, float* out_val_acc, const gb_fit_stop* stop,
                     float* best_params, int32_t* out_epochs, int32_t* out_best_epoch, const gb_optimizer* opt,
                     const gb_dense_reg* reg, const gb_dense_dropout* drop, void* stream) {
  GB_REQUIRE(!split || out_val_loss, GB_E_ARG, "split needs out_val_loss");
  GB_REQUIRE(!split || val_batch >= 1, GB_E_ARG, "val_batch=%d must be >= 1", val_batch);
  GB_REQUIRE(!stop || (best_params && out_epochs && out_best_epoch), GB_E_ARG,
             "stop needs best_params, out_epochs and out_best_epoch");
  GB_REQUIRE(!stop || gb::aligned16(best_params), GB_E_ARG, "best_params must be 16-byte aligned");
  bool any = false, any_drop = false;
  const int rc = gb_fit::check_reg_drop(net, reg, drop, any, any_drop);
  if (rc != GB_OK) return rc;
  const FitEntry entry = stop ? FIT_STOP : split ? FIT_SPLIT : FIT_PLAIN;
  return launch_fit(net, params, adam_m, adam_v, jobs, split, n_jobs, max_rows, x, y, row_map, perm, hp, split ? val_batch : 1,
                    out_loss, out_acc, out_val_loss, out_val_acc, stop, best_params, out_epochs, out_best_epoch, entry, opt,
                    any ? reg : nullptr, any_drop ? drop : nullptr, stream);
}

int gb_ffae_fit_reg(const gb_ffnet* net, float* params, float* adam_m, float* adam_v, const gb_job* jobs,
                    const gb_fit_split* split, int32_t n_jobs, int32_t max_rows, const float* x, const float* y,
                    const int32_t* row_map, const int32_t* perm, const gb_fit_hparams* hp, int32_t val_batch,
                    float* out_loss, float* out_acc, float* out_val_loss, float* out_val_acc, const gb_fit_stop* stop,
                    float* best_params, int32_t* out_epochs, int32_t* out_best_epoch, const gb_optimizer* opt,
                    const gb_dense_reg* reg, void* stream) {
  return gb_ffae_fit_drop(net, params, adam_m, adam_v, jobs, split, n_jobs, max_rows, x, y, row_map, perm, hp, val_batch, out_loss,
                          out_acc, out_val_loss, out_val_acc, stop, best_params, out_epochs, out_best_epoch, opt, reg, nullptr, stream);
}

int gb_ffae_fit_opt(const gb_ffnet* net, float* params, float* adam_m, float* adam_v, const gb_job* jobs,
                    const gb_fit_split* split, int32_t n_jobs, int32_t max_rows, const float* x, const float* y,
                    const int32_t* row_map, const int32_t* perm, const gb_fit_hparams* hp, int32_t val_batch,
                    float* out_loss, float* out_acc, float* out_val_loss, float* out_val_acc, const gb_fit_stop* stop,
                    float* best_params, int32_t* out_epochs, int32_t* out_best_epoch, const gb_optimizer* opt, void* stream) {
  return gb_ffae_fit_reg(net, params, adam_m, adam_v, jobs, split, n_jobs, max_rows, x, y, row_map, perm, hp, val_batch, out_loss,
                         out_acc, out_val_loss, out_val_acc, stop, best_params, out_epochs, out_best_epoch, opt, nullptr, stream);
}

}  // extern "C"

// defined after the entry points: the tag nvcc gives this file's anonymous namespace follows its first external definition, and
// the kernels' names carry that tag
namespace gb_fit {

int check_fit(const gb_ffnet* net, float* params, float* adam_m, float* adam_v, const gb_job* jobs, const float* x, const float* y,
              const int32_t* perm, const gb_fit_hparams* hp, float* out_loss, const gb_optimizer* opt) {
  int rc = gb::validate_ffnet(net);
  if (rc != GB_OK) return rc;
  rc = gb::validate_optimizer(opt);
  if (rc != GB_OK) return rc;
  GB_REQUIRE(params && adam_m && adam_v && jobs && x && y && hp && out_loss, GB_E_ARG,
             "params/adam_m/adam_v/jobs/x/y/hp/out_loss must be non-NULL");
  GB_REQUIRE(hp->epochs >= 1, GB_E_ARG, "epochs=%d must be >= 1", hp->epochs);
  GB_REQUIRE(hp->batch_size >= 1, GB_E_ARG, "batch_size=%d must be >= 1", hp->batch_size);
  GB_REQUIRE(hp->shuffle >= 0 && hp->shuffle <= 2, GB_E_ARG, "shuffle=%d unknown", hp->shuffle);
  GB_REQUIRE(hp->shuffle != 2 || perm, GB_E_ARG, "shuffle=2 needs perm");
  GB_REQUIRE(hp->loss >= GB_LOSS_MSE && hp->loss <= GB_LOSS_LOG_COSH, GB_E_ARG, "loss=%d unknown (gb_loss: 0..5)", hp->loss);
  GB_REQUIRE(gb::aligned16(params) && gb::aligned16(adam_m) && gb::aligned16(adam_v) && gb::aligned16(x) &&
                 gb::aligned16(y),
             GB_E_ALIGN, "params/adam/x/y must be 16-byte aligned");
  return GB_OK;
}

int check_split_stop(const gb_fit_split* split, int32_t val_batch, const float* out_val_loss, const gb_fit_stop* stop,
                     const int32_t* out_epochs, const int32_t* out_best_epoch) {
  GB_REQUIRE(!split || out_val_loss, GB_E_ARG, "split needs out_val_loss");
  GB_REQUIRE(!split || val_batch >= 1, GB_E_ARG, "val_batch=%d must be >= 1", val_batch);
  GB_REQUIRE(!stop || (out_epochs && out_best_epoch), GB_E_ARG, "stop needs best_params, out_epochs and out_best_epoch");
  return GB_OK;
}

int check_best_params(const gb_fit_stop* stop, const float* best_params) {
  GB_REQUIRE(!stop || best_params, GB_E_ARG, "stop needs best_params, out_epochs and out_best_epoch");
  GB_REQUIRE(!stop || gb::aligned16(best_params), GB_E_ARG, "best_params must be 16-byte aligned");
  return GB_OK;
}

int check_reg_drop(const gb_ffnet* net, const gb_dense_reg* reg, const gb_dense_dropout* drop, bool& any_reg, bool& any_drop) {
  any_reg = false;  // a record of zeros is no record: the kernels of gb_ffae_fit_opt
  if (reg != nullptr) {
    const int rc = gb::validate_ffnet(net);
    if (rc != GB_OK) return rc;
    auto ok = [](float v) { return v >= 0.f && v < 3.0e38f; };  // false for NaN and inf
    const struct { const char* name; const float* c; } fields[] = {
        {"kernel_l1", reg->kernel_l1}, {"kernel_l2", reg->kernel_l2}, {"bias_l1", reg->bias_l1}, {"bias_l2", reg->bias_l2}};
    for (const auto& f : fields)
      for (int l = 0; l < net->n_layers; ++l) {
        GB_REQUIRE(ok(f.c[l]), GB_E_ARG, "reg %s[%d]=%g must be finite and >= 0", f.name, l, (double)f.c[l]);
        any_reg = any_reg || f.c[l] != 0.f;
      }
  }
  any_drop = false;  // likewise: all-zero rates run the kernels of gb_ffae_fit_reg
  if (drop != nullptr) {
    const int rc = gb::validate_ffnet(net);
    if (rc != GB_OK) return rc;
    for (int l = 0; l < GB_MAX_LAYERS; ++l) {
      const float r = drop->rate[l];
      GB_REQUIRE(r >= 0.f && r < 1.f, GB_E_ARG, "dropout rate[%d]=%g must be finite, >= 0 and < 1", l, (double)r);  // false for NaN
      GB_REQUIRE(r == 0.f || l < net->n_layers, GB_E_ARG, "dropout rate[%d]=%g: the net has %d layers (rate[l] is on the input of layer l)",
                 l, (double)r, net->n_layers);
      GB_REQUIRE(r == 0.f || l == 0 || net->l1[l - 1] == 0.f, GB_E_ARG,
                 "dropout rate[%d]=%g on the output of layer %d, which has an activity L1: not supported", l, (double)r, l - 1);
      any_drop = any_drop || r != 0.f;
    }
  }
  return GB_OK;
}

FitFamily fit_family(const gb_fit_hparams* hp, const gb_optimizer* opt, const gb_dense_reg* reg, const gb_dense_dropout* drop) {
  if (drop != nullptr) return FAMILY_DROP;
  if (reg != nullptr) return FAMILY_REG;
  if (!gb::plain_adam(opt)) return FAMILY_OPT;
  return hp->loss == GB_LOSS_MSE ? FAMILY_MSE : FAMILY_LOSS;
}

int setup_fit(const gb_ffnet* net, float* params, float* adam_m, float* adam_v, const gb_job* jobs, const gb_fit_split* split,
              int32_t max_rows, const float* x, const float* y, const int32_t* row_map, const int32_t* perm, const gb_fit_hparams* hp,
              int32_t val_batch, float* out_loss, float* out_acc, float* out_val_loss, float* out_val_acc, const gb_fit_stop* stop,
              float* best_params, int32_t* out_epochs, int32_t* out_best_epoch, const gb_optimizer* opt, const gb_dense_reg* reg,
              const gb_dense_dropout* drop, FitArgs& a, bool& w_global, size_t& smem) {
  a = FitArgs{};
  smem = 0;
  w_global = false;
  int rc = plan_fit(net, a, w_global, smem);
  if (rc != GB_OK) return rc;
  a.hp = *hp;
  const bool use_opt = !gb::plain_adam(opt);
  if (opt != nullptr && !use_opt) {  // plain Adam runs the Adam kernels, from the optimizer's hyperparameters
    a.hp.lr = opt->lr; a.hp.beta1 = opt->beta1; a.hp.beta2 = opt->beta2; a.hp.eps = opt->eps;
  }
  if (use_opt) a.opt = *opt;
  if (reg != nullptr || drop != nullptr) {  // the REG and DROP kernels are OPT kernels: plain Adam, too, runs through gb::opt_update there
    if (reg != nullptr) a.reg = *reg;  // else zeros: the DROP kernels add a penalty of 0
    if (opt != nullptr) {
      a.opt = *opt;
    } else {
      a.opt = gb_optimizer{};
      a.opt.kind = GB_OPT_ADAM; a.opt.lr = hp->lr; a.opt.beta1 = hp->beta1; a.opt.beta2 = hp->beta2; a.opt.eps = hp->eps;
    }
  }
  if (drop != nullptr) {
    for (int l = 0; l < GB_MAX_LAYERS; ++l) {
      if (drop->rate[l] == 0.f) continue;
      const double r = (double)drop->rate[l];
      a.drop_layers |= 1u << l;
      a.drop_thr[l] = (uint32_t)floor(r * 4294967296.0);
      a.drop_scale[l] = (float)(1.0 / (1.0 - r));
    }
  }
  const int L = net->n_layers;
  a.max_rows = max_rows;
  a.pstride = (long)gb_ffnet_param_stride(net);
  a.sstride = (long)gb_ffae_fit_state_stride(net);
  a.gather_layer = 0;
  for (int l = 1; l < L; ++l)
    if (a.im.np[l] <= a.im.np[a.gather_layer]) a.gather_layer = l;  // the last of the narrowest layers
  a.gather_layer2 = a.gather_layer;
  for (int l = 0, best = 1 << 30; l < L; ++l)
    if (l != a.gather_layer && a.im.np[l] < best) { best = a.im.np[l]; a.gather_layer2 = l; }  // the narrowest of the others
  a.params = params; a.adam_m = adam_m; a.adam_v = adam_v; a.jobs = jobs; a.x = x; a.y = y; a.perm = perm;
  a.out_loss = out_loss; a.out_acc = out_acc;
  a.split = split; a.row_map = row_map; a.val_batch = val_batch; a.out_val_loss = out_val_loss; a.out_val_acc = out_val_acc;
  a.stop = stop; a.best_params = best_params; a.out_epochs = out_epochs; a.out_best_epoch = out_best_epoch;
  return GB_OK;
}

}  // namespace gb_fit
