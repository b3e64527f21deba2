// Shared by the two LSTM fit families (lstm_fit.cu, lstm_fit_tc.cu): the capture of one optimizer step as a CUDA graph, and
// Keras' EarlyStopping inside the fit launch (gb_lstm_fit_stop, gb_lstm_fit_tc_stop).
//
// The rule's state lives on the device, after the fit's own workspace (gb_lstm_fit_stop_state_bytes): per job a copy of its
// gb_job, then a State record, then the count of live jobs.  The step kernels read the job copies in place of the caller's
// array.  When a job stops, its copy's n_rows becomes 0, so the step kernels' job_batch gives it no windows from then on: it
// does no work and its optimizer step count stays where it is, without any change to those kernels.  Once every job has
// stopped the step graph skips its body: the body is an `if` node whose condition a one-thread head kernel sets from the live
// count, so each remaining replay runs two tiny kernels (the step's window setter and that head).
#pragma once
#include <math_constants.h>

#include "gb_common.cuh"

namespace {
namespace lstm_stop {

struct State {
  gb_fit_stop rule;  // the job's record, copied from the caller's host array
  float best;        // best monitored value (+-inf before the first improvement); a float32 history entry, so a float holds it
  int32_t wait;      // epochs since the last improvement that also beat the baseline
  int32_t snap;      // the epoch just ended goes to best_params
  int32_t stopped;
};
static_assert(sizeof(gb_job) == 24 && sizeof(State) == 56, "stop state layout");

inline size_t state_bytes(int n_jobs) { return (size_t)n_jobs * (sizeof(gb_job) + sizeof(State)) + 16; }

// The caller's records, validated on the host: nothing is enqueued for a bad one.
inline int validate(const gb_fit_stop* stop, int n_jobs) {
  for (int j = 0; j < n_jobs; ++j) {
    const gb_fit_stop& r = stop[j];
    GB_REQUIRE(r.monitor >= 0 && r.monitor <= 3, GB_E_ARG, "stop[%d].monitor=%d unknown (0 loss, 1 accuracy, 2 val_loss, 3 val_accuracy)", j,
               r.monitor);
    GB_REQUIRE(r.mode == 1 || r.mode == -1, GB_E_ARG, "stop[%d].mode=%d must be +1 or -1", j, r.mode);
    GB_REQUIRE(r.patience >= 0, GB_E_ARG, "stop[%d].patience=%d must be >= 0", j, r.patience);
    GB_REQUIRE(r.min_delta >= 0.0, GB_E_ARG, "stop[%d].min_delta=%g must be >= 0", j, r.min_delta);
  }
  return GB_OK;
}

// Records reach the device as kernel parameters, REC per launch: a copy from pageable host memory could wait for the stream.
constexpr int REC = 96;  // 96 * 40 bytes + the header stay inside the 4 KB parameter space
struct Records {
  int j0, n;
  gb_fit_stop rec[REC];
};

__global__ void init_kernel(const Records r, const gb_job* jobs, int n_jobs, int epochs, gb_job* job_copy, State* st, int* live,
                            int32_t* out_epochs, int32_t* out_best_epoch) {
  const int i = threadIdx.x, j = r.j0 + i;
  if (r.j0 == 0 && i == 0) *live = n_jobs;
  if (i >= r.n) return;
  job_copy[j] = jobs[j];
  State s;
  s.rule = r.rec[i];
  s.best = s.rule.mode > 0 ? CUDART_INF_F : -CUDART_INF_F;
  s.wait = 0;
  s.snap = 0;
  s.stopped = 0;
  st[j] = s;
  out_epochs[j] = epochs;  // rewritten by an early stop
  out_best_epoch[j] = -1;
}

// The end of epoch `epoch`.  For a live job: its history entries, as the families' epoch kernels write them, then the rule on
// the monitored entry (keras 3 EarlyStopping.on_epoch_end; models.py EarlyStopping.update), in double as gb_ffae_fit_stop
// compares.  The LSTM fit reports loss and accuracy only: a val_* monitor is unavailable, so such a job never stops and takes no
// snapshot.  A stopped job's history entries are left as they are.  The epoch sums are reset for every job.
__global__ void epoch_kernel(const gb_job* jobs, int n_jobs, gb_job* job_copy, State* st, int* live, float* loss_sum, float* hit_sum,
                             float* out_loss, float* out_acc, int32_t* out_epochs, int32_t* out_best_epoch, int epoch, int epochs) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n_jobs) return;
  State s = st[j];
  const float ls = loss_sum[j], hs = hit_sum[j];
  loss_sum[j] = 0.f;
  hit_sum[j] = 0.f;
  s.snap = 0;
  if (!s.stopped) {
    const float n = (float)max(jobs[j].n_rows, 1);
    const long h = (long)j * epochs + epoch;
    out_loss[h] = ls / n;
    out_acc[h] = hs / n;
    const gb_fit_stop& rule = s.rule;
    if (rule.monitor <= 1 && epoch >= rule.start_from_epoch) {
      const float v = rule.monitor == 0 ? ls / n : hs / n;
      auto improves = [&](double x, double ref) -> bool { return rule.mode > 0 ? x + rule.min_delta < ref : x - rule.min_delta > ref; };
      int best_epoch = out_best_epoch[j];
      if (rule.restore_best && best_epoch < 0) {
        s.snap = 1;
        best_epoch = epoch;
      }
      ++s.wait;
      if (improves(v, s.best)) {
        s.best = v;
        best_epoch = epoch;
        if (rule.restore_best) s.snap = 1;
        if (!rule.has_baseline || improves(v, rule.baseline)) s.wait = 0;
      } else if (s.wait >= rule.patience && epoch > 0) {
        s.stopped = 1;
        job_copy[j].n_rows = 0;
        out_epochs[j] = epoch + 1;
        atomicSub(live, 1);
      }
      out_best_epoch[j] = best_epoch;
    }
  }
  st[j] = s;
}

// grid (chunks, n_jobs): the slot of every job whose snapshot flag is set goes params -> best_params (restore = 0); at the end
// of the call, the snapshot of every job with restore_best and a snapshot goes back (restore = 1).  Other CTAs exit at once.
__global__ void __launch_bounds__(256) copy_kernel(const gb_job* jobs, const State* st, const int32_t* out_best_epoch, float* params,
                                                   float* best_params, long pstride, long n_params, int restore) {
  const int j = blockIdx.y;
  if (restore ? !(st[j].rule.restore_best && out_best_epoch[j] >= 0) : !st[j].snap) return;
  const long base = (long)jobs[j].slot * pstride;
  const float* src = restore ? best_params + base : params + base;
  float* dst = restore ? params + base : best_params + base;
  for (long i = (long)blockIdx.x * 256 + threadIdx.x; i < n_params; i += (long)gridDim.x * 256) dst[i] = src[i];
}

__global__ void cond_kernel(cudaGraphConditionalHandle handle, const int* live) { cudaGraphSetConditional(handle, *live > 0 ? 1u : 0u); }

// graph = [cond_kernel] -> [if (live > 0) body]; *body is owned by the conditional node
inline cudaError_t conditional_graph(cudaGraph_t* graph, cudaGraph_t* body, const int* live) {
  cudaError_t ce = cudaGraphCreate(graph, 0);
  if (ce != cudaSuccess) return ce;
  cudaGraphConditionalHandle handle;
  if ((ce = cudaGraphConditionalHandleCreate(&handle, *graph, 0, 0)) != cudaSuccess) return ce;
  void* args[] = {&handle, &live};
  cudaKernelNodeParams kp{};
  kp.func = reinterpret_cast<void*>(cond_kernel);
  kp.gridDim = dim3(1);
  kp.blockDim = dim3(1);
  kp.kernelParams = args;
  cudaGraphNode_t head, cond;
  if ((ce = cudaGraphAddKernelNode(&head, *graph, nullptr, 0, &kp)) != cudaSuccess) return ce;
  cudaGraphNodeParams np{};
  np.type = cudaGraphNodeTypeConditional;
  np.conditional.handle = handle;
  np.conditional.type = cudaGraphCondTypeIf;
  np.conditional.size = 1;
  if ((ce = cudaGraphAddNode(&cond, *graph, &head, 1, &np)) != cudaSuccess) return ce;
  *body = np.conditional.phGraph_out[0];
  return cudaSuccess;
}

// The rule's device state for one call, laid out after `ws_bytes` of fit workspace, and the launches around the steps.
struct Run {
  const gb_job* jobs;
  int n_jobs, epochs;
  gb_job* job_copy;
  State* st;
  int* live;
  int32_t *out_epochs, *out_best_epoch;
  float *params, *best_params;
  long pstride, n_params;

  Run(void* workspace, size_t ws_bytes, const gb_job* jobs_, int n_jobs_, int epochs_, int32_t* out_epochs_, int32_t* out_best_epoch_,
      float* params_, float* best_params_, long pstride_, long n_params_)
      : jobs(jobs_), n_jobs(n_jobs_), epochs(epochs_), out_epochs(out_epochs_), out_best_epoch(out_best_epoch_), params(params_),
        best_params(best_params_), pstride(pstride_), n_params(n_params_) {
    job_copy = reinterpret_cast<gb_job*>(static_cast<char*>(workspace) + ws_bytes);  // ws_bytes is a multiple of 8
    st = reinterpret_cast<State*>(job_copy + n_jobs);
    live = reinterpret_cast<int*>(st + n_jobs);
  }
  void init(const gb_fit_stop* stop, cudaStream_t s) const {
    Records r;
    for (r.j0 = 0; r.j0 < n_jobs; r.j0 += REC) {
      r.n = min(REC, n_jobs - r.j0);
      for (int i = 0; i < r.n; ++i) r.rec[i] = stop[r.j0 + i];
      init_kernel<<<1, REC, 0, s>>>(r, jobs, n_jobs, epochs, job_copy, st, live, out_epochs, out_best_epoch);
    }
  }
  void end_epoch(int epoch, float* loss_sum, float* hit_sum, float* out_loss, float* out_acc, cudaStream_t s) const {
    epoch_kernel<<<(n_jobs + 127) / 128, 128, 0, s>>>(jobs, n_jobs, job_copy, st, live, loss_sum, hit_sum, out_loss, out_acc, out_epochs,
                                                      out_best_epoch, epoch, epochs);
    copy(0, s);
  }
  void finish(cudaStream_t s) const { copy(1, s); }
  void copy(int restore, cudaStream_t s) const {
    copy_kernel<<<dim3((unsigned)((n_params + 256 * 8 - 1) / (256 * 8)), n_jobs), 256, 0, s>>>(jobs, st, out_best_epoch, params, best_params,
                                                                                             pstride, n_params, restore);
  }
};

}  // namespace lstm_stop

// One optimizer step's launch sequence, record(stream), captured once and instantiated for replay.  live NULL: the launches are
// the graph.  Otherwise they are the body of an `if` node that runs only while *live > 0; GB_E_CUDA if the runtime cannot
// build that node (there is no unconditional fall-back).
template <class Record>
int capture_step(cudaGraphExec_t* gexec, const int* live, Record record) {
  cudaGraph_t graph = nullptr;
  cudaStream_t cap = nullptr;  // the caller's stream may be the legacy default stream, which cannot capture
  GB_CUDA_CHECK(cudaStreamCreateWithFlags(&cap, cudaStreamNonBlocking));
  {
    cudaError_t ce;
    const char* what = "cudaStreamBeginCapture";
    if (live != nullptr) {
      cudaGraph_t body = nullptr;
      ce = lstm_stop::conditional_graph(&graph, &body, live);
      what = "building the conditional node of the LSTM optimizer step";
      if (ce == cudaSuccess) {
        ce = cudaStreamBeginCaptureToGraph(cap, body, nullptr, nullptr, 0, cudaStreamCaptureModeThreadLocal);
        what = "cudaStreamBeginCaptureToGraph";
      }
    } else {
      ce = cudaStreamBeginCapture(cap, cudaStreamCaptureModeThreadLocal);
    }
    if (ce != cudaSuccess) {
      cudaStreamDestroy(cap);
      if (graph != nullptr) cudaGraphDestroy(graph);
      gb::set_error("%s failed: %s", what, cudaGetErrorString(ce));
      return GB_E_CUDA;
    }
  }
  record(cap);  // everything recorded, not run
  {
    cudaGraph_t captured = nullptr;
    const cudaError_t ce = cudaStreamEndCapture(cap, &captured);
    cudaStreamDestroy(cap);
    if (ce != cudaSuccess || captured == nullptr) {
      if (graph != nullptr) cudaGraphDestroy(graph);
      gb::set_error("capturing the LSTM optimizer step failed: %s", cudaGetErrorString(ce));
      return GB_E_CUDA;
    }
    if (graph == nullptr) graph = captured;  // with a conditional node, `captured` is its body
  }
  {
    const cudaError_t ce = cudaGraphInstantiate(gexec, graph, 0);
    cudaGraphDestroy(graph);
    if (ce != cudaSuccess) {
      gb::set_error("cudaGraphInstantiate failed: %s", cudaGetErrorString(ce));
      return GB_E_CUDA;
    }
  }
  return GB_OK;
}

}  // namespace
