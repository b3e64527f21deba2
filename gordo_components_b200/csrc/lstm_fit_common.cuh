// Shared by the two LSTM fit families (lstm_fit.cu on fp32 CUDA cores, lstm_fit_tc.cu on the tensor cores): the launch
// arguments and workspace layout, the kernels that do not depend on how the GEMMs are tiled (gate gradients, optimizer, step
// bookkeeping), Keras' EarlyStopping inside the fit launch (gb_lstm_fit_stop, gb_lstm_fit_tc_stop), the capture of one
// optimizer step as a CUDA graph, and the host driver of a whole fit (fit_driver).  A family adds its forward, head,
// input-gradient and weight-gradient kernels and a small policy that records them.
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

struct Lay {
  int in, u;       // input width, units
  int act;
  long kofs;       // offset of [K; U] (rows in + u, 4u columns) in the parameter vector; bias follows
  long zofs, cofs, hofs, dhofs, nxofs;  // workspace offsets (floats, per job): gates [L][Bp][4u], c / h [L][Bp][u], dh_seq [L][Bp][u], (dh_next, dc_next) [2][Bp][u]
};

// The fields up to `opt` are the fp32 family's; the tensor-core family's follow, so that adding them moved no parameter of the
// fp32 kernels.
struct FitArgs {
  int n_layers, L, F, T_out, out_act, lookahead;
  Lay lay[GB_MAX_LAYERS];
  long dofs;        // Dense kernel offset in the parameter vector
  long pstride, ws_stride;  // floats per slot / per job
  long gofs;        // gradient vector offset in the job workspace
  long topdh;       // [Bp][u_top] dh of the last LSTM layer at t = L-1
  float* params;
  float *adam_m, *adam_v;
  int* adam_t;
  const gb_job* jobs;
  const float *x, *y;
  float* ws;
  float *loss_sum, *hit_sum;  // [n_jobs]
  const int* step;            // device: {first window, nominal batch size} of the optimizer step being replayed (the launch
                              // sequence of one step is captured once as a CUDA graph; only these two numbers change)
  float lr, b1, b2, eps;
  int loss;                   // gb_loss of the head
  gb_optimizer opt;           // another optimizer than plain Adam (lstm_opt_kernel)
  int Bp;                     // batch rows the workspace holds per timestep
  long doutofs;               // tensor-core head: [Bp][T_out] d(loss)/d(Dense pre-activation)
  long partofs;               // tensor-core head: [Bp / head_rows][2] loss and hit sums per head slice
};

__device__ __forceinline__ float sigm(float z) { return 1.f / (1.f + expf(-z)); }
__device__ __forceinline__ int job_batch(const gb_job& job, int win0, int bsz) { return max(0, min(bsz, job.n_rows - win0)); }

// Workspace layout of one job (floats) for batches of up to Bp windows; returns the total.  head_rows > 0 adds the tensor-core
// head's areas: the loss gradient and the partial sums of its head_rows-row slices.
inline long layout(const gb_lstmnet* net, int Bp, int head_rows, FitArgs* a) {
  long ofs = 0, pofs = 0;
  int in = net->n_features;
  const long L = net->lookback;
  a->Bp = Bp;
  for (int l = 0; l < net->n_layers; ++l) {
    const int u = net->units[l];
    Lay& ly = a->lay[l];
    ly.in = in; ly.u = u; ly.act = net->act[l];
    ly.kofs = pofs;
    pofs += 4L * u * (in + u + 1);
    ly.zofs = ofs; ofs += L * Bp * 4 * u;
    ly.cofs = ofs; ofs += L * Bp * u;
    ly.hofs = ofs; ofs += L * Bp * u;
    ly.dhofs = ofs; ofs += (l + 1 < net->n_layers) ? L * Bp * u : 0;
    ly.nxofs = ofs; ofs += 2L * Bp * u;
    in = u;
  }
  a->dofs = pofs;
  a->topdh = ofs; ofs += (long)Bp * in;
  if (head_rows > 0) {
    a->doutofs = ofs; ofs += (long)Bp * net->n_features_out;
    a->partofs = ofs; ofs += 2L * (Bp / head_rows);
  }
  a->gofs = ofs; ofs += (long)gb_lstm_param_stride(net);
  return (ofs + 3) / 4 * 4;
}

// Bytes of a fit's workspace: the jobs' areas, then the epoch's loss and hit sums per job and the step's two numbers.
inline size_t workspace_bytes(long ws_stride, int n_jobs) { return (size_t)(ws_stride * n_jobs + 2L * n_jobs + 4) * sizeof(float); }

// ---------------------------------------------------------------------------------------------- backward: gate gradients
// grid (ceil(Bp*u/256), n_jobs).  Overwrites the saved gates of (l, t) with dz, updates dc_next.
__global__ void __launch_bounds__(256) lstm_bwd_gates_kernel(const FitArgs a, int l, int t) {
  const gb_job job = a.jobs[blockIdx.y];
  const int nb = job_batch(job, a.step[0], a.step[1]);
  if (nb == 0) return;
  const Lay ly = a.lay[l];
  const int u = ly.u, u4 = 4 * u, Bp = a.Bp;
  const int i = blockIdx.x * 256 + threadIdx.x;
  const int b = i / u, un = i - b * u;
  if (b >= nb) return;
  float* ws = a.ws + (long)blockIdx.y * a.ws_stride;
  float* Z = ws + ly.zofs + (long)t * Bp * u4 + (long)b * u4;
  const float ig = Z[un], fg = Z[u + un], gg = Z[2 * u + un], og = Z[3 * u + un];
  const long bu = (long)b * u + un;
  const float c = ws[ly.cofs + (long)t * Bp * u + bu];
  const float cp = t > 0 ? ws[ly.cofs + (long)(t - 1) * Bp * u + bu] : 0.f;
  float* nx = ws + ly.nxofs;  // dh_next [Bp][u], dc_next [Bp][u]
  const bool last_t = t == a.L - 1;
  float dh = last_t ? 0.f : nx[bu];
  if (l == a.n_layers - 1) {
    if (last_t) dh += ws[a.topdh + bu];
  } else {
    dh += ws[ly.dhofs + (long)t * Bp * u + bu];
  }
  const float ac = gb::apply_act(ly.act, c);
  const float dc = dh * og * gb::act_grad_from_output(ly.act, ac) + (last_t ? 0.f : nx[(long)Bp * u + bu]);
  Z[un] = dc * gg * ig * (1.f - ig);
  Z[u + un] = dc * cp * fg * (1.f - fg);
  Z[2 * u + un] = dc * ig * gb::act_grad_from_output(ly.act, gg);
  Z[3 * u + un] = dh * ac * og * (1.f - og);
  nx[(long)Bp * u + bu] = dc * fg;
}

// ---------------------------------------------------------------------------------------------- Adam
//   m += (g-m)(1-b1); v += (g^2-v)(1-b2); w -= lr sqrt(1-b2^t)/(1-b1^t) m/(sqrt(v)+eps)   [3P keras]
__global__ void __launch_bounds__(256) lstm_adam_kernel(const FitArgs a, long n_params) {
  const gb_job job = a.jobs[blockIdx.y];
  if (job_batch(job, a.step[0], a.step[1]) == 0) return;
  const int t = a.adam_t[job.slot] + 1;
  const float alpha = (float)((double)a.lr * sqrt(1.0 - pow((double)a.b2, (double)t)) / (1.0 - pow((double)a.b1, (double)t)));
  const float* G = a.ws + (long)blockIdx.y * a.ws_stride + a.gofs;
  float* P = a.params + (long)job.slot * a.pstride;
  float* M = a.adam_m + (long)job.slot * a.pstride;
  float* V = a.adam_v + (long)job.slot * a.pstride;
  for (long i = (long)blockIdx.x * 256 + threadIdx.x; i < n_params; i += (long)gridDim.x * 256) {
    const float g = G[i];
    const float m = M[i] + (g - M[i]) * (1.f - a.b1);
    const float v = V[i] + (g * g - V[i]) * (1.f - a.b2);
    M[i] = m;
    V[i] = v;
    P[i] -= alpha * m / (sqrtf(v) + a.eps);
  }
}
// Every other optimizer than plain Adam (gb::opt_update; state slots 0 / 1 = adam_m / adam_v), captured in place of lstm_adam_kernel.
// The per-step scalars come from the slot's step count, once per CTA (for Nadam a product over the slot's steps, a few cycles each).
__global__ void __launch_bounds__(256) lstm_opt_kernel(const FitArgs a, long n_params) {
  const gb_job job = a.jobs[blockIdx.y];
  if (job_batch(job, a.step[0], a.step[1]) == 0) return;
  __shared__ gb::OptStep s_st;
  if (threadIdx.x == 0) s_st = gb::opt_step_at(a.opt, a.adam_t[job.slot] + 1);
  __syncthreads();
  const gb::OptStep st = s_st;
  const float* G = a.ws + (long)blockIdx.y * a.ws_stride + a.gofs;
  float* P = a.params + (long)job.slot * a.pstride;
  float* S0 = a.adam_m + (long)job.slot * a.pstride;
  float* S1 = a.adam_v + (long)job.slot * a.pstride;
  for (long i = (long)blockIdx.x * 256 + threadIdx.x; i < n_params; i += (long)gridDim.x * 256) {
    float w = P[i], s0 = S0[i], s1 = S1[i];
    gb::opt_update(a.opt, st, w, G[i], s0, s1);
    P[i] = w;
    S0[i] = s0;
    S1[i] = s1;
  }
}
__global__ void lstm_bump_kernel(const FitArgs a, int n_jobs) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n_jobs && job_batch(a.jobs[j], a.step[0], a.step[1]) > 0) a.adam_t[a.jobs[j].slot] += 1;
}
__global__ void lstm_set_step_kernel(int* step, int win0, int bsz) {
  step[0] = win0;
  step[1] = bsz;
}
// epoch bookkeeping: history[job][epoch] = sums / n_windows; sums reset
__global__ void lstm_epoch_kernel(const gb_job* jobs, int n_jobs, float* loss_sum, float* hit_sum, float* out_loss, float* out_acc, int epoch, int epochs) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n_jobs) return;
  if (epoch >= 0) {
    const float n = (float)max(jobs[j].n_rows, 1);
    out_loss[(long)j * epochs + epoch] = loss_sum[j] / n;
    out_acc[(long)j * epochs + epoch] = hit_sum[j] / n;
  }
  loss_sum[j] = 0.f;
  hit_sum[j] = 0.f;
}

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

// One fit call of a family (gb_lstm_fit_opt / _stop, gb_lstm_fit_tc_opt / _stop; stop NULL: no rule, the step graph and
// launches as they have always been).  The family policy supplies
//   max_batch, who          the largest batch_size it takes, and its name in the refusal of a larger one;
//   rows(batch_size)        the batch rows of its workspace (FitArgs::Bp);  head_rows  as for layout();
//   prepare(a)              its set-up before the first launch (shared-memory limits), returning a gb_status;
//   record(a, n_jobs, s)    the launches of one step up to the weight gradients; the optimizer and step count follow here.
template <class Family>
int fit_driver(Family fam, const gb_lstmnet* net, float* params, float* adam_m, float* adam_v, int32_t* adam_t, const gb_job* jobs,
               int32_t n_jobs, int32_t max_windows, const float* x, const float* y, const gb_lstm_fit_hparams* hp, void* workspace,
               float* out_loss, float* out_acc, int32_t loss, const gb_optimizer* opt, const gb_fit_stop* stop, float* best_params,
               int32_t* out_epochs, int32_t* out_best_epoch, void* stream) {
  int rc = gb::validate_lstmnet(net);
  if (rc != GB_OK) return rc;
  if ((rc = gb::validate_optimizer(opt)) != GB_OK) return rc;
  GB_REQUIRE(loss >= GB_LOSS_MSE && loss <= GB_LOSS_LOG_COSH, GB_E_ARG, "loss=%d unknown (gb_loss: 0..5)", loss);
  GB_REQUIRE(params && adam_m && adam_v && adam_t && jobs && x && y && hp && workspace && out_loss && out_acc, GB_E_ARG, "NULL argument");
  GB_REQUIRE(n_jobs >= 0 && n_jobs <= 65535 && max_windows >= 0, GB_E_ARG, "bad n_jobs/max_windows");
  GB_REQUIRE(hp->epochs >= 0 && hp->batch_size >= 1, GB_E_ARG, "epochs=%d batch_size=%d", hp->epochs, hp->batch_size);
  GB_REQUIRE(hp->batch_size <= Family::max_batch, GB_E_SHAPE, "batch_size=%d: %s handles batches of at most %d windows", hp->batch_size,
             Family::who, Family::max_batch);
  GB_REQUIRE(hp->lookahead >= 0, GB_E_ARG, "Value of `lookahead` can not be negative, is %d", hp->lookahead);
  if (stop != nullptr) {
    GB_REQUIRE(best_params && out_epochs && out_best_epoch, GB_E_ARG, "stop needs best_params, out_epochs and out_best_epoch");
    GB_REQUIRE(gb::aligned16(best_params), GB_E_ARG, "best_params must be 16-byte aligned");
    if ((rc = lstm_stop::validate(stop, n_jobs)) != GB_OK) return rc;
  }
  if (n_jobs == 0) return GB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  FitArgs a{};
  a.n_layers = net->n_layers; a.L = net->lookback; a.F = net->n_features; a.T_out = net->n_features_out; a.out_act = net->out_act;
  a.lookahead = hp->lookahead;
  a.ws_stride = layout(net, Family::rows(hp->batch_size), Family::head_rows, &a);
  a.pstride = (long)gb_lstm_param_stride(net);
  a.params = params; a.adam_m = adam_m; a.adam_v = adam_v; a.adam_t = adam_t; a.jobs = jobs; a.x = x; a.y = y;
  a.ws = static_cast<float*>(workspace);
  a.loss_sum = a.ws + a.ws_stride * n_jobs;
  a.hit_sum = a.loss_sum + n_jobs;
  a.lr = hp->lr; a.b1 = hp->beta1; a.b2 = hp->beta2; a.eps = hp->eps;
  const bool use_opt = !gb::plain_adam(opt);
  if (opt != nullptr && !use_opt) { a.lr = opt->lr; a.b1 = opt->beta1; a.b2 = opt->beta2; a.eps = opt->eps; }  // plain Adam: the Adam kernel
  if (use_opt) a.opt = *opt;
  a.loss = loss;
  const long n_params = (long)gb_lstm_param_count(net);
  if ((rc = fam.prepare(a)) != GB_OK) return rc;
  const int jb = (n_jobs + 127) / 128;

  int* d_step = reinterpret_cast<int*>(a.hit_sum + n_jobs);
  a.step = d_step;
  const lstm_stop::Run run(workspace, workspace_bytes(a.ws_stride, n_jobs), jobs, n_jobs, hp->epochs, out_epochs, out_best_epoch, params,
                           best_params, a.pstride, n_params);
  if (stop != nullptr) {
    run.init(stop, st);
    a.jobs = run.job_copy;  // a job that stops gets n_rows 0 here, so job_batch gives it no windows
  }
  // One optimizer step is thousands of small launches (18 per timestep for the fp32 family): captured once as a CUDA graph and
  // replayed per step, the step's (first window, batch size) being read from device memory -- launch overhead was >90 % of a
  // step for few machines.
  cudaGraphExec_t gexec = nullptr;
  rc = capture_step(&gexec, stop != nullptr ? run.live : nullptr, [&](cudaStream_t s) {
    fam.record(a, n_jobs, s);
    const dim3 grid((unsigned)((n_params + 256 * 8 - 1) / (256 * 8)), n_jobs);
    if (use_opt) lstm_opt_kernel<<<grid, 256, 0, s>>>(a, n_params);
    else lstm_adam_kernel<<<grid, 256, 0, s>>>(a, n_params);
    lstm_bump_kernel<<<jb, 128, 0, s>>>(a, n_jobs);
  });
  if (rc != GB_OK) return rc;
  auto step = [&](int win0, int bsz) -> int {
    lstm_set_step_kernel<<<1, 1, 0, st>>>(d_step, win0, bsz);
    const cudaError_t ce = cudaGraphLaunch(gexec, st);
    if (ce != cudaSuccess) {
      gb::set_error("cudaGraphLaunch failed: %s", cudaGetErrorString(ce));
      return GB_E_CUDA;
    }
    return GB_OK;
  };
  auto train = [&]() -> int {
    lstm_epoch_kernel<<<jb, 128, 0, st>>>(jobs, n_jobs, a.loss_sum, a.hit_sum, out_loss, out_acc, -1, hp->epochs);
    if (hp->primer) {
      if ((rc = step(0, 1)) != GB_OK) return rc;
      lstm_epoch_kernel<<<jb, 128, 0, st>>>(jobs, n_jobs, a.loss_sum, a.hit_sum, out_loss, out_acc, -1, hp->epochs);
    }
    for (int e = 0; e < hp->epochs; ++e) {
      for (int w = 0; w < max_windows; w += hp->batch_size)
        if ((rc = step(w, hp->batch_size)) != GB_OK) return rc;
      if (stop != nullptr) run.end_epoch(e, a.loss_sum, a.hit_sum, out_loss, out_acc, st);
      else lstm_epoch_kernel<<<jb, 128, 0, st>>>(jobs, n_jobs, a.loss_sum, a.hit_sum, out_loss, out_acc, e, hp->epochs);
    }
    if (stop != nullptr) run.finish(st);
    return GB_OK;
  };
  rc = train();
  cudaGraphExecDestroy(gexec);  // the enqueued replays keep what they need
  if (rc != GB_OK) return rc;
  GB_CUDA_CHECK(cudaGetLastError());
  return GB_OK;
}

}  // namespace
