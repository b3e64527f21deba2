// The Dense fit kernels with Keras Dropout (gb_ffae_fit_drop): the nine ffae_fit_drop_kernel<WG, DG, SPLIT, STOP> instantiations,
// one per (memory plan group, entry point), in an object of their own.  launch_fit (ffae_fit.cu) plans the fit, fills the record
// and hands it here; see ffae_fit_kernels.cuh for the kernels and include/gordo_b200.h (gb_dense_dropout) for what they compute.
#include "ffae_fit_kernels.cuh"

namespace gb_fit {

int launch_drop(const FitArgs& a, FitEntry entry, bool w_global, size_t smem, int n_jobs, cudaStream_t stream) {
  auto launch = [&](auto kernel) -> int {
    GB_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kernel<<<n_jobs, THREADS, smem, stream>>>(a);
    return GB_OK;
  };
  if (entry == FIT_STOP) {
    if (a.d_global > 0) return launch(ffae_fit_drop_kernel<true, true, true, true>);
    if (w_global) return launch(ffae_fit_drop_kernel<true, false, true, true>);
    return launch(ffae_fit_drop_kernel<false, false, true, true>);
  }
  if (entry == FIT_SPLIT) {
    if (a.d_global > 0) return launch(ffae_fit_drop_kernel<true, true, true, false>);
    if (w_global) return launch(ffae_fit_drop_kernel<true, false, true, false>);
    return launch(ffae_fit_drop_kernel<false, false, true, false>);
  }
  if (a.d_global > 0) return launch(ffae_fit_drop_kernel<true, true, false, false>);
  if (w_global) return launch(ffae_fit_drop_kernel<true, false, false, false>);
  return launch(ffae_fit_drop_kernel<false, false, false, false>);
}

}  // namespace gb_fit
