// K3, variant 1: LSTM autoencoder prediction on the fp32 CUDA cores, fused over layers and timesteps.
//
// Replaces KerasLSTMBaseEstimator.predict (gordo/machine/model/models.py:618-660) for the stacks of
// factories/lstm_autoencoder.py:72-103 without materialising windows (models.py:713-793): output row j of a job
// is the network applied to x rows [x_row + j, x_row + j + lookback).  One CTA advances a block of BW windows one
// timestep at a time through *all* LSTM layers (layer l at step t needs only h_{l-1,t} and its own (h,c)_{t-1}), so
// the only state is the current h and c of every layer, resident in shared memory -- no [windows][lookback][units]
// sequence ever exists.  Weights (keras layout kernel [in][4u] | recurrent_kernel [u][4u] | bias [4u], gates i,f,c,o)
// stream from L2; lanes run along units so every weight load is one coalesced segment and the activations of the
// window block are shared-memory broadcasts.
#include "gb_common.cuh"

namespace {

constexpr int THREADS = 256;
constexpr int NWARPS = THREADS / 32;
constexpr int BW = 16;  // windows per CTA

struct LstmArgs {
  gb_lstmnet net;
  int hofs[GB_MAX_LAYERS];    // offset of layer l's h block (floats) inside the h (and c) state area
  int hpitch[GB_MAX_LAYERS];  // row pitch of layer l's state block
  long kofs[GB_MAX_LAYERS];   // offset of layer l's kernel in the slot's parameter vector
  long dofs;                  // offset of the Dense kernel
  int state_floats;           // floats of one state area (h or c)
  int tmp_pitch, x_pitch;
  long pstride;
  const float* params;
  const gb_job* jobs;
  const float* x;
  float* out;
};

__device__ __forceinline__ float sigmoidf_(float z) { return 1.f / (1.f + expf(-z)); }

// one LSTM layer, one timestep, WPT windows per thread (windows [w0, w0+WPT)), unit = ublock*32 + lane
template <int WPT>
__device__ __forceinline__ void lstm_cell_step(const float* __restrict__ Kw, const float* __restrict__ Uw,
                                               const float* __restrict__ bw, const float* in_vec, int in_pitch, int n_inp,
                                               const float* h_own, float* c_own, int s_pitch, float* h_tmp, int tmp_pitch,
                                               int u, int act, int task) {
  const int lane = threadIdx.x & 31;
  const int wgroups = BW / WPT;
  const int ublock = task / wgroups, w0 = (task - ublock * wgroups) * WPT;
  const int unit = ublock * 32 + lane;
  const bool live = unit < u;
  const int uu = live ? unit : 0;
  const int u4 = 4 * u;
  float acc[WPT][4];
#pragma unroll
  for (int g = 0; g < 4; ++g) {
    const float b = live ? __ldg(bw + g * u + uu) : 0.f;
#pragma unroll
    for (int w = 0; w < WPT; ++w) acc[w][g] = b;
  }
  // z += in_vec . kernel ; z += h_own . recurrent_kernel
#pragma unroll 1
  for (int part = 0; part < 2; ++part) {
    const float* W = part == 0 ? Kw : Uw;
    const float* vec = part == 0 ? in_vec : h_own;
    const int pitch = part == 0 ? in_pitch : s_pitch;
    const int kdim = part == 0 ? n_inp : u;
    const int k4 = kdim & ~3;
    for (int k = 0; k < k4; k += 4) {
      float kw[4][4];
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)
#pragma unroll
        for (int g = 0; g < 4; ++g) kw[kk][g] = live ? __ldg(W + (long)(k + kk) * u4 + g * u + uu) : 0.f;
#pragma unroll
      for (int w = 0; w < WPT; ++w) {
        const float4 av = *reinterpret_cast<const float4*>(vec + (w0 + w) * pitch + k);
#pragma unroll
        for (int g = 0; g < 4; ++g) {
          acc[w][g] = fmaf(av.x, kw[0][g], acc[w][g]);
          acc[w][g] = fmaf(av.y, kw[1][g], acc[w][g]);
          acc[w][g] = fmaf(av.z, kw[2][g], acc[w][g]);
          acc[w][g] = fmaf(av.w, kw[3][g], acc[w][g]);
        }
      }
    }
    for (int k = k4; k < kdim; ++k) {
      float kw[4];
#pragma unroll
      for (int g = 0; g < 4; ++g) kw[g] = live ? __ldg(W + (long)k * u4 + g * u + uu) : 0.f;
#pragma unroll
      for (int w = 0; w < WPT; ++w) {
        const float av = vec[(w0 + w) * pitch + k];
#pragma unroll
        for (int g = 0; g < 4; ++g) acc[w][g] = fmaf(av, kw[g], acc[w][g]);
      }
    }
  }
  if (live) {
#pragma unroll
    for (int w = 0; w < WPT; ++w) {
      const float ig = sigmoidf_(acc[w][0]), fg = sigmoidf_(acc[w][1]), og = sigmoidf_(acc[w][3]);
      const float cc = fg * c_own[(w0 + w) * s_pitch + unit] + ig * gb::apply_act(act, acc[w][2]);
      c_own[(w0 + w) * s_pitch + unit] = cc;
      h_tmp[(w0 + w) * tmp_pitch + unit] = og * gb::apply_act(act, cc);
    }
  }
}

__global__ void __launch_bounds__(THREADS) lstm_infer_kernel(const LstmArgs a) {
  extern __shared__ __align__(16) float smem[];
  float* hs = smem;
  float* cs = hs + a.state_floats;
  float* tmp = cs + a.state_floats;
  float* xs = tmp + BW * a.tmp_pitch;

  const gb_job job = a.jobs[blockIdx.y];
  const int wbase = blockIdx.x * BW;
  if (wbase >= job.n_rows) return;
  const int nwin = min(BW, job.n_rows - wbase);
  const int tid = threadIdx.x, warp = tid >> 5;
  const int F = a.net.n_features, NL = a.net.n_layers, LB = a.net.lookback;
  const float* P = a.params + (long)job.slot * a.pstride;

  for (int i = tid; i < 2 * a.state_floats + BW * a.tmp_pitch + BW * a.x_pitch; i += THREADS) smem[i] = 0.f;
  __syncthreads();

  for (int t = 0; t < LB; ++t) {
    // x rows of this timestep: window w reads row x_row + wbase + w + t
    for (int idx = tid; idx < BW * F; idx += THREADS) {
      const int w = idx / F, f = idx - w * F;
      xs[w * a.x_pitch + f] = (w < nwin) ? __ldg(a.x + (job.x_row + wbase + w + t) * (long)F + f) : 0.f;
    }
    __syncthreads();
    for (int l = 0; l < NL; ++l) {
      const int u = a.net.units[l];
      const int n_inp = (l == 0) ? F : a.net.units[l - 1];
      const float* in_vec = (l == 0) ? xs : hs + a.hofs[l - 1];
      const int in_pitch = (l == 0) ? a.x_pitch : a.hpitch[l - 1];
      const float* Kw = P + a.kofs[l];
      const float* Uw = Kw + (long)n_inp * 4 * u;
      const float* bw = Uw + (long)u * 4 * u;
      float* h_own = hs + a.hofs[l];
      float* c_own = cs + a.hofs[l];
      const int ublocks = (u + 31) / 32;
      // choose the window split so that every warp has work when the layer is narrow
      int wpt = BW;
      while (wpt > 2 && ublocks * (BW / wpt) < NWARPS) wpt >>= 1;
      const int tasks = ublocks * (BW / wpt);
      for (int task = warp; task < tasks; task += NWARPS) {
        switch (wpt) {
          case 16: lstm_cell_step<16>(Kw, Uw, bw, in_vec, in_pitch, n_inp, h_own, c_own, a.hpitch[l], tmp, a.tmp_pitch, u, a.net.act[l], task); break;
          case 8: lstm_cell_step<8>(Kw, Uw, bw, in_vec, in_pitch, n_inp, h_own, c_own, a.hpitch[l], tmp, a.tmp_pitch, u, a.net.act[l], task); break;
          case 4: lstm_cell_step<4>(Kw, Uw, bw, in_vec, in_pitch, n_inp, h_own, c_own, a.hpitch[l], tmp, a.tmp_pitch, u, a.net.act[l], task); break;
          default: lstm_cell_step<2>(Kw, Uw, bw, in_vec, in_pitch, n_inp, h_own, c_own, a.hpitch[l], tmp, a.tmp_pitch, u, a.net.act[l], task); break;
        }
      }
      __syncthreads();  // every read of h_{l,t-1} is done
      for (int idx = tid; idx < BW * u; idx += THREADS) {
        const int w = idx / u, j = idx - w * u;
        h_own[w * a.hpitch[l] + j] = tmp[w * a.tmp_pitch + j];
      }
      __syncthreads();
    }
  }
  // Dense head on the last layer's final hidden state
  {
    const int u = a.net.units[NL - 1], n_out = a.net.n_features_out;
    const float* hl = hs + a.hofs[NL - 1];
    const int hp = a.hpitch[NL - 1];
    const float* Wd = P + a.dofs;
    const float* bd = Wd + (long)u * n_out;
    for (int idx = tid; idx < nwin * n_out; idx += THREADS) {
      const int w = idx / n_out, j = idx - w * n_out;
      float acc = __ldg(bd + j);
      for (int k = 0; k < u; ++k) acc = fmaf(hl[w * hp + k], __ldg(Wd + (long)k * n_out + j), acc);
      a.out[(job.out_row + wbase + w) * (long)n_out + j] = gb::apply_act(a.net.out_act, acc);
    }
  }
}

int pitch4(int w) {
  int p4 = (w + 3) / 4;
  if ((p4 & 1) == 0) ++p4;
  return 4 * p4;
}

}  // namespace

extern "C" {

size_t gb_lstm_param_count(const gb_lstmnet* net) {
  if (gb::validate_lstmnet(net) != GB_OK) return 0;
  size_t p = 0;
  int in = net->n_features;
  for (int l = 0; l < net->n_layers; ++l) {
    const size_t u = net->units[l];
    p += 4 * u * (in + u + 1);
    in = (int)u;
  }
  return p + (size_t)in * net->n_features_out + net->n_features_out;
}

size_t gb_lstm_param_stride(const gb_lstmnet* net) { return (gb_lstm_param_count(net) + 3) / 4 * 4; }

size_t gb_lstm_workspace_bytes(const gb_lstmnet*, int32_t, int32_t) { return 0; }

int gb_lstm_infer(const gb_lstmnet* net, const float* params, const gb_job* jobs, int32_t n_jobs, int32_t max_rows,
                  const float* x, float* out_model, void* /*workspace*/, void* stream) {
  int rc = gb::validate_lstmnet(net);
  if (rc != GB_OK) return rc;
  GB_REQUIRE(params && jobs && x && out_model, GB_E_ARG, "params/jobs/x/out_model must be non-NULL");
  GB_REQUIRE(n_jobs >= 0 && max_rows >= 0, GB_E_ARG, "bad n_jobs/max_rows");
  if (n_jobs == 0 || max_rows == 0) return GB_OK;
  LstmArgs a{};
  a.net = *net;
  int ofs = 0, maxu = 0;
  long pofs = 0;
  int in = net->n_features;
  for (int l = 0; l < net->n_layers; ++l) {
    const int u = net->units[l];
    a.hpitch[l] = pitch4(u);
    a.hofs[l] = ofs;
    ofs += BW * a.hpitch[l];
    a.kofs[l] = pofs;
    pofs += 4L * u * (in + u + 1);
    in = u;
    maxu = max(maxu, u);
  }
  a.dofs = pofs;
  a.state_floats = ofs;
  a.tmp_pitch = pitch4(maxu);
  a.x_pitch = pitch4(net->n_features);
  a.pstride = (long)gb_lstm_param_stride(net);
  a.params = params; a.jobs = jobs; a.x = x; a.out = out_model;
  const size_t smem = (size_t)(2 * a.state_floats + BW * a.tmp_pitch + BW * a.x_pitch) * sizeof(float);
  GB_REQUIRE(smem <= 227 * 1024, GB_E_SMEM, "LSTM stack needs %zu bytes of shared memory for its state", smem);
  GB_CUDA_CHECK(cudaFuncSetAttribute(lstm_infer_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int blocks = (max_rows + BW - 1) / BW;
  for (int j0 = 0; j0 < n_jobs; j0 += 65535) {  // gridDim.y carries the job index: larger fleets go out as several launches
    a.jobs = jobs + j0;
    lstm_infer_kernel<<<dim3(blocks, n_jobs - j0 < 65535 ? n_jobs - j0 : 65535), THREADS, smem, (cudaStream_t)stream>>>(a);
  }
  GB_CUDA_CHECK(cudaGetLastError());
  return GB_OK;
}

}  // extern "C"
