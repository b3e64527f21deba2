// The grouped Dense fit (gb_ffae_fit_group): the jobs of several architectures that share a memory plan in one launch.
//
// The fit runs one persistent CTA per job and keeps the job's network in that CTA's shared memory (ffae_fit.cu), so nothing ties
// the CTAs of a launch to one architecture but the launch record.  Here every group has its own FitArgs, filled by the same
// setup_fit as a per-net launch with the group's net and pointers; the records and the job -> group map are copied to the caller's
// device workspace together, and each CTA reads its group's record through L1 (the body's `a`).  The body is ffae_fit_body.cuh, the template flags
// are those of the per-net kernel of the same family, and the plan is a template flag, so a job computes exactly what it computes in
// a per-net launch of its group.  The record is not staged in shared memory: the static arrays stay those the plans reserve
// FIT_STATIC_SMEM for, so every net the per-net fit takes can join a group.  The kernels live in an object of their own, so that
// ffae_fit.o and ffae_fit_drop.o keep exactly the kernels they had.
#include <cstring>
#include <string>
#include <vector>
#include "ffae_fit_kernels.cuh"

namespace {

using gb_fit::FIT_PLAIN;
using gb_fit::FIT_SPLIT;
using gb_fit::FIT_STOP;
using gb_fit::FitEntry;

template <bool WG, bool DG, bool SPLIT, bool STOP, bool LOSS, bool OPT, bool REG, bool DROP>
__global__ void __launch_bounds__(THREADS, 1) ffae_fit_group_kernel(const FitArgs* __restrict__ groups, const int32_t* __restrict__ job_group) {
  const FitArgs& a = groups[job_group[blockIdx.x]];
#include "ffae_fit_body.cuh"
}

// the last error, prefixed with the group it concerns
int group_error(int rc, int g) {
  const std::string msg = gb_last_error();
  gb::set_error("group %d: %s", g, msg.c_str());
  return rc;
}

// the workspace: the records, then the job -> group map
size_t workspace_bytes(int32_t n_groups, int32_t n_jobs) {
  return (size_t)(n_groups > 0 ? n_groups : 0) * sizeof(FitArgs) + (size_t)(n_jobs > 0 ? n_jobs : 0) * sizeof(int32_t);
}

}  // namespace

extern "C" size_t gb_ffae_fit_group_workspace_bytes(int32_t n_groups, int32_t n_jobs) { return workspace_bytes(n_groups, n_jobs); }

extern "C" int gb_ffae_fit_group(const gb_fit_group* groups, int32_t n_groups, const int32_t* job_group, const gb_job* jobs,
                                 const gb_fit_split* split, int32_t n_jobs, int32_t max_rows, const int32_t* row_map,
                                 const int32_t* perm, const gb_fit_hparams* hp, int32_t val_batch, float* out_loss, float* out_acc,
                                 float* out_val_loss, float* out_val_acc, const gb_fit_stop* stop, int32_t* out_epochs,
                                 int32_t* out_best_epoch, const gb_optimizer* opt, const gb_dense_reg* reg,
                                 const gb_dense_dropout* drop, void* workspace, void* stream) {
  GB_REQUIRE(n_groups >= 1, GB_E_ARG, "n_groups=%d must be >= 1", n_groups);
  GB_REQUIRE(groups != nullptr, GB_E_ARG, "groups must be non-NULL");
  GB_REQUIRE(workspace != nullptr && gb::aligned16(workspace), GB_E_ARG,
             "workspace must be non-NULL and 16-byte aligned (gb_ffae_fit_group_workspace_bytes)");
  GB_REQUIRE(n_jobs >= 0 && max_rows >= 0, GB_E_ARG, "n_jobs=%d and max_rows=%d must be >= 0", n_jobs, max_rows);
  GB_REQUIRE(n_jobs == 0 || job_group != nullptr, GB_E_ARG, "job_group must be non-NULL");
  int rc = gb_fit::check_split_stop(split, val_batch, out_val_loss, stop, out_epochs, out_best_epoch);
  if (rc != GB_OK) return rc;
  // every group is checked as gb_ffae_fit_drop checks its one net; the family reg and drop select must be the same for all
  bool any_reg = false, any_drop = false;
  for (int g = 0; g < n_groups; ++g) {
    const gb_fit_group& G = groups[g];
    bool r = false, d = false;
    rc = gb_fit::check_best_params(stop, G.best_params);
    if (rc == GB_OK) rc = gb_fit::check_reg_drop(&G.net, reg, drop, r, d);
    if (rc == GB_OK) rc = gb_fit::check_fit(&G.net, G.params, G.adam_m, G.adam_v, jobs, G.x, G.y, perm, hp, out_loss, opt);
    if (rc != GB_OK) return group_error(rc, g);
    if (g == 0) { any_reg = r; any_drop = d; }
    GB_REQUIRE(r == any_reg && d == any_drop, GB_E_ARG,
               "group %d: reg / dropout are %s / %s on its layers but %s / %s on group 0's: the groups would run different kernel families",
               g, r ? "non-zero" : "zero", d ? "non-zero" : "zero", any_reg ? "non-zero" : "zero", any_drop ? "non-zero" : "zero");
  }
  for (int j = 0; j < n_jobs; ++j)
    GB_REQUIRE(job_group[j] >= 0 && job_group[j] < n_groups, GB_E_ARG, "job_group[%d]=%d outside [0, %d)", j, job_group[j], n_groups);
  if (n_jobs == 0 || max_rows == 0) return GB_OK;
  if (!any_reg) reg = nullptr;
  if (!any_drop) drop = nullptr;

  std::vector<FitArgs> args(n_groups);
  bool w_global = false;
  size_t smem = 0;
  for (int g = 0; g < n_groups; ++g) {
    const gb_fit_group& G = groups[g];
    bool wg = false;
    size_t sm = 0;
    rc = gb_fit::setup_fit(&G.net, G.params, G.adam_m, G.adam_v, jobs, split, max_rows, G.x, G.y, row_map, perm, hp,
                           split ? val_batch : 1, out_loss, out_acc, out_val_loss, out_val_acc, stop, G.best_params, out_epochs,
                           out_best_epoch, opt, reg, drop, args[g], wg, sm);
    if (rc != GB_OK) return group_error(rc, g);
    if (g == 0) w_global = wg;
    GB_REQUIRE(wg == w_global && args[g].d_global == args[0].d_global, GB_E_ARG,
               "group %d: memory plan (weights in L2 %d, dz buffers in L2 %d) differs from group 0's (%d, %d)", g, (int)wg,
               args[g].d_global, (int)w_global, args[0].d_global);
    smem = sm > smem ? sm : smem;
  }

  const size_t rec_bytes = (size_t)n_groups * sizeof(FitArgs);
  std::vector<unsigned char> host(workspace_bytes(n_groups, n_jobs));
  memcpy(host.data(), args.data(), rec_bytes);
  memcpy(host.data() + rec_bytes, job_group, (size_t)n_jobs * sizeof(int32_t));
  const cudaStream_t st = (cudaStream_t)stream;
  // a copy from pageable memory: it has been staged when the call returns, so `host` may go
  GB_CUDA_CHECK(cudaMemcpyAsync(workspace, host.data(), host.size(), cudaMemcpyHostToDevice, st));
  const FitArgs* d_args = static_cast<const FitArgs*>(workspace);
  const int32_t* d_group = reinterpret_cast<const int32_t*>(static_cast<unsigned char*>(workspace) + rec_bytes);
  auto launch = [&](auto kernel) -> int {
    GB_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kernel<<<n_jobs, THREADS, smem, st>>>(d_args, d_group);
    return GB_OK;
  };
  const FitEntry entry = stop ? FIT_STOP : split ? FIT_SPLIT : FIT_PLAIN;
  const int d_global = args[0].d_global;
  auto dispatch = [&](auto loss, auto opt_, auto reg_, auto drop_) -> int {
    constexpr bool LS = decltype(loss)::value, OP = decltype(opt_)::value, RG = decltype(reg_)::value, DR = decltype(drop_)::value;
    if (entry == FIT_STOP) {
      if (d_global > 0) return launch(ffae_fit_group_kernel<true, true, true, true, LS, OP, RG, DR>);
      if (w_global) return launch(ffae_fit_group_kernel<true, false, true, true, LS, OP, RG, DR>);
      return launch(ffae_fit_group_kernel<false, false, true, true, LS, OP, RG, DR>);
    }
    if (entry == FIT_SPLIT) {
      if (d_global > 0) return launch(ffae_fit_group_kernel<true, true, true, false, LS, OP, RG, DR>);
      if (w_global) return launch(ffae_fit_group_kernel<true, false, true, false, LS, OP, RG, DR>);
      return launch(ffae_fit_group_kernel<false, false, true, false, LS, OP, RG, DR>);
    }
    if (d_global > 0) return launch(ffae_fit_group_kernel<true, true, false, false, LS, OP, RG, DR>);
    if (w_global) return launch(ffae_fit_group_kernel<true, false, false, false, LS, OP, RG, DR>);
    return launch(ffae_fit_group_kernel<false, false, false, false, LS, OP, RG, DR>);
  };
  const std::false_type no{};
  const std::true_type yes{};
  int rc2 = GB_OK;
  switch (gb_fit::fit_family(hp, opt, reg, drop)) {  // the per-net launch's family, so the arithmetic is the same code
    case gb_fit::FAMILY_DROP: rc2 = dispatch(yes, yes, yes, yes); break;
    case gb_fit::FAMILY_REG: rc2 = dispatch(yes, yes, yes, no); break;
    case gb_fit::FAMILY_OPT: rc2 = dispatch(yes, yes, no, no); break;
    case gb_fit::FAMILY_LOSS: rc2 = dispatch(yes, no, no, no); break;
    default: rc2 = dispatch(no, no, no, no);
  }
  if (rc2 != GB_OK) return rc2;
  GB_CUDA_CHECK(cudaGetLastError());
  return GB_OK;
}
