// Body of the Dense fit kernels (ffae_fit.cu): included inside ffae_fit_kernel, ffae_fit_reg_kernel and ffae_fit_drop_kernel, where
// the template flags WG, DG, SPLIT, STOP, LOSS, OPT, REG and DROP, THREADS / NWARPS / BR, FitArgs a and the helpers of ffae_fit.cu
// are in scope.  Not a header of its own: see the description of the flags above the three kernels.
  extern __shared__ __align__(16) float smem[];
  __shared__ float s_red[3][NWARPS];
  __shared__ float s_alpha[2];  // Adam step size of optimizer step t at [t & 1]: written one step ahead, off the critical path
  __shared__ std::conditional_t<OPT, gb::OptStep, float> s_opt[2];  // OPT: the same for the optimizer's per-step scalars
  __shared__ int s_idx[2][BR];
  __shared__ long long s_phase[2 * GB_MAX_LAYERS + 4];

  const int job_id = blockIdx.x;
  const gb_job job = a.jobs[job_id];
  const int n = job.n_rows;
  const bool stopping = STOP && a.stop != nullptr;
  if (n <= 0) {
    if (stopping && threadIdx.x == 0) { a.out_epochs[job_id] = 0; a.out_best_epoch[job_id] = -1; }
    return;
  }
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int L = a.net.n_layers, n_in = a.n_in, n_out = a.n_out;
  const bool tracing = a.trace != nullptr && blockIdx.x == 0 && tid == 0;
  long long t_mark = 0;
  if (tracing) {
    for (int i = 0; i < 2 * GB_MAX_LAYERS + 4; ++i) s_phase[i] = 0;
    t_mark = clock64();
  }
  auto stamp = [&](int phase) {  // called by everyone right after a barrier; one thread books the cycles since the previous stamp
    if (tracing) { const long long now = clock64(); s_phase[phase] += now - t_mark; t_mark = now; }
  };
  const int B = a.hp.batch_size;
  float* P = a.params + (long)job.slot * a.pstride;
  float* Mg = a.adam_m + (long)job.slot * a.sstride;
  float* sW = WG ? Mg + 2 * a.wfloats : smem;
  float* Vg = a.adam_v + (long)job.slot * a.sstride;

  // ---- weights -> padded smem image; zero every staging buffer ------------------------------------
  for (int i = tid; i < a.smem_floats; i += THREADS) smem[i] = 0.f;
  if (WG)
    for (int i = tid; i < a.wfloats; i += THREADS) sW[i] = 0.f;  // the padding of the image must read as zero
  __syncthreads();
  float pen = 0.f;  // REG: this thread's share of the weight penalty of the current weights
  for (int l = 0; l < L; ++l) {
    const int K = a.net.dims[l], N = a.net.dims[l + 1], Np = a.im.np[l];
    const float* Wg = P + a.im.pofs[l];
    float* dst = sW + a.im.wofs[l];
    for (int idx = tid; idx < K * N; idx += THREADS) {
      const int k = idx / N, nn = idx - k * N;
      dst[k * Np + nn] = Wg[idx];
      if constexpr (REG) pen += a.reg.kernel_l1[l] * fabsf(Wg[idx]) + a.reg.kernel_l2[l] * (Wg[idx] * Wg[idx]);
    }
    for (int nn = tid; nn < N; nn += THREADS) {
      sW[a.im.bofs[l] + nn] = Wg[K * N + nn];
      if constexpr (REG) pen += a.reg.bias_l1[l] * fabsf(Wg[K * N + nn]) + a.reg.bias_l2[l] * (Wg[K * N + nn] * Wg[K * N + nn]);
    }
  }

  const float* xbase = a.x + job.x_row * (long)n_in;
  const float* ybase = a.y + job.x_row * (long)n_out;
  const int steps = (n + B - 1) / B;
  int nv = 0;           // held-out positions
  long map_ofs = -1;
  if (SPLIT && a.split != nullptr) {
    nv = a.split[job_id].n_val;
    if (a.row_map != nullptr) map_ofs = a.split[job_id].map_ofs;
  }
  const int VB = a.val_batch;
  const int vsteps = SPLIT && nv > 0 ? (nv + VB - 1) / VB : 0;  // mini-batches s in [steps, steps + vsteps) are held-out ones
  auto held_out = [&](int s) -> bool { return SPLIT && s >= steps; };
  auto batch_rows = [&](int s) -> int { return held_out(s) ? min(VB, nv - (s - steps) * VB) : min(B, n - s * B); };
  const uint32_t key_base = mix32((uint32_t)a.hp.seed ^ mix32((uint32_t)(a.hp.seed >> 32) + 0x632be5abU * (uint32_t)(job.slot + 1)));
  const uint32_t drop_key = DROP ? mix32(key_base ^ 0x2545f491U) : 0u;  // DROP: the job's dropout key (gb_dense_dropout)

  auto row_index = [&](int e, int i) -> int {
    if (a.hp.shuffle == 0) return i;
    if (a.hp.shuffle == 2) return a.perm[((long)job_id * a.hp.epochs + e) * a.max_rows + i];
    return (int)permute_index((uint32_t)i, (uint32_t)n, mix32(key_base + (uint32_t)e * 0x9e3779b9U));
  };
  // row (relative to x_row) of row i of mini-batch s of epoch e
  auto batch_row = [&](int e, int s, int i) -> int {
    if (!SPLIT) return row_index(e, s * B + i);
    const int p = held_out(s) ? n + (s - steps) * VB + i : row_index(e, s * B + i);
    return map_ofs >= 0 ? a.row_map[map_ofs + p] : p;
  };
  // rows [r_lo, r_hi) of chunk c (32 rows) of mini-batch s of epoch e, by n_warps warps
  auto gather = [&](int buf, int e, int s, int c, int first_warp, int n_warps, int r_lo = 0, int r_hi = BR) {
    const int nb = min(BR, batch_rows(s) - c * BR);
    float* xs = smem + a.xofs[buf];
    float* ys = smem + a.yofs[buf];
    for (int r = r_lo + warp - first_warp; r < min(nb, r_hi); r += n_warps) {
      const int src = s_idx[buf][r];
      const float* xr = xbase + (long)src * n_in;
      const float* yr = ybase + (long)src * n_out;
      if ((n_in & 3) == 0) {
        for (int c = lane * 4; c < n_in; c += 128) __pipeline_memcpy_async(xs + r * a.apitch[0] + c, xr + c, 16);
      } else {
        for (int c = lane; c < n_in; c += 32) __pipeline_memcpy_async(xs + r * a.apitch[0] + c, xr + c, 4);
      }
      if ((n_out & 3) == 0) {
        for (int c = lane * 4; c < n_out; c += 128) __pipeline_memcpy_async(ys + r * a.ypitch + c, yr + c, 16);
      } else {
        for (int c = lane; c < n_out; c += 32) __pipeline_memcpy_async(ys + r * a.ypitch + c, yr + c, 4);
      }
    }
    __pipeline_commit();
  };

  const float omb1 = 1.f - a.hp.beta1, omb2 = 1.f - a.hp.beta2, eps = a.hp.eps;
  int t_step = a.hp.step0;
  int cur = 0;
  // the visiting order is resolved one chunk ahead of its gather by the last warp (a row per lane): the keyed permutation costs a
  // few hundred instructions per row, which every warp would otherwise repeat in front of its cp.async
  auto advance = [&](int& e, int& s, int& c) -> bool {  // next chunk in visiting order; false past the last epoch
    const int nch = (batch_rows(s) + BR - 1) / BR;
    if (++c == nch) { c = 0; if (++s == steps + vsteps) { s = 0; ++e; } }
    return e < a.hp.epochs;
  };
  auto stage_indices = [&](int buf, int e, int s, int c) {
    const int nb = min(BR, batch_rows(s) - c * BR);
    if (lane < nb) s_idx[buf][lane] = batch_row(e, s, c * BR + lane);
  };
  auto adam_alpha = [&](int t_int) -> float {  // lr * sqrt(1 - b2^t) / (1 - b1^t)
    const double t = (double)t_int;
    return (float)((double)a.hp.lr * sqrt(1.0 - pow((double)a.hp.beta2, t)) / (1.0 - pow((double)a.hp.beta1, t)));
  };
  if constexpr (OPT) {
    if (tid == 0) s_opt[(t_step + 1) & 1] = gb::opt_step_at(a.opt, t_step + 1);
  } else {
    if (tid == 0) s_alpha[(t_step + 1) & 1] = adam_alpha(t_step + 1);
  }
  if (warp == NWARPS - 1) {
    int e1 = 0, s1 = 0, c1 = 0;
    stage_indices(0, 0, 0, 0);
    if (advance(e1, s1, c1)) stage_indices(1, e1, s1, c1);
  }
  __syncthreads();
  stamp(2 * L + 2);  // set-up
  gather(0, 0, 0, 0, 0, NWARPS);
  float* Gacc = Mg + a.wfloats;  // gradient sums of a multi-chunk mini-batch (same padded layout as the weights)
  // dz buffer b: shared memory, or -- for stacks whose activations leave no room (256-wide encoders) -- the unused part of the slot's
  // Adam-v state area (the second and third third of it), which stays in L2
  auto dz_buf = [&](int b) -> float* {
    if (!DG) return smem + a.dofs[b];
    return b < 3 - a.d_global ? smem + a.dofs[b] : Vg + a.wfloats + (long)(b - (3 - a.d_global)) * BR * a.dpitch;
  };

  // ---- epoch statistics (keras History: sample-weighted mean of the per-batch total loss) -------------
  auto epoch_stats = [&](float v0, float v1, float v2, float* out_l, float* out_a, int rows, int e) {
    for (int o = 16; o > 0; o >>= 1) {
      v0 += __shfl_xor_sync(0xffffffffu, v0, o);
      v1 += __shfl_xor_sync(0xffffffffu, v1, o);
      v2 += __shfl_xor_sync(0xffffffffu, v2, o);
    }
    if (lane == 0) { s_red[0][warp] = v0; s_red[1][warp] = v1; s_red[2][warp] = v2; }
    __syncthreads();
    if (tid == 0) {
      float q0 = 0.f, q1 = 0.f, q2 = 0.f;
      for (int w = 0; w < NWARPS; ++w) { q0 += s_red[0][w]; q1 += s_red[1][w]; q2 += s_red[2][w]; }
      out_l[(long)job_id * a.hp.epochs + e] = (q0 / (float)n_out + q1) / (float)rows;
      if (out_a) out_a[(long)job_id * a.hp.epochs + e] = q2 / (float)rows;
    }
    __syncthreads();
  };

  // ---- the weight image in canonical layout (the slot's parameter vector), by every thread -----------------
  auto write_image = [&](float* dst) {
    for (int l = 0; l < L; ++l) {
      const int K = a.net.dims[l], N = a.net.dims[l + 1], Np = a.im.np[l];
      float* Wg = dst + a.im.pofs[l];
      const float* src = sW + a.im.wofs[l];
      for (int idx = tid; idx < K * N; idx += THREADS) {
        const int k = idx / N, nn = idx - k * N;
        Wg[idx] = src[k * Np + nn];
      }
      for (int nn = tid; nn < N; nn += THREADS) Wg[K * N + nn] = sW[a.im.bofs[l] + nn];
    }
  };

  // ---- EarlyStopping (keras 3 EarlyStopping.on_epoch_end, models.py EarlyStopping.update) ------------------------------
  // Thread 0 owns the state, three registers across the epoch loop: the record is re-read from global memory at each epoch's
  // end.  `best` is +-inf or a monitored float32 value, so a float holds it exactly; with restore_best a snapshot exists once
  // an epoch has counted, i.e. when best_epoch >= 0.
  float best = stopping && a.stop[job_id].mode > 0 ? CUDART_INF_F : -CUDART_INF_F;
  int wait = 0, best_epoch = -1;
  if (stopping && tid == 0) a.out_epochs[job_id] = a.hp.epochs;  // rewritten by an early stop

  for (int e = 0; e < a.hp.epochs; ++e) {
    float acc_sq = 0.f, acc_reg = 0.f, acc_hit = 0.f;
    for (int s = 0; s < steps + vsteps; ++s) {
      const bool val = held_out(s);               // forward only: loss statistics, no optimizer step
      if (val && s == steps) {                    // the training statistics are complete: the held-out ones start from zero
        epoch_stats(acc_sq, acc_reg, acc_hit, a.out_loss, a.out_acc, n, e);
        acc_sq = acc_reg = acc_hit = 0.f;
      }
      const int nbt = batch_rows(s);              // rows of this mini-batch
      const int nchunks = (nbt + BR - 1) / BR;
      if (!val) ++t_step;
      if constexpr (REG) acc_reg += (float)nbt * pen;  // the penalty of the weights this mini-batch's forward pass uses
     for (int c = 0; c < nchunks; ++c) {
      const int nb = min(BR, nbt - c * BR);        // rows of this chunk
      const bool first_chunk = c == 0, last_chunk = c + 1 == nchunks;
      // ---- prefetch the next chunk, then wait for the current one ------------------------
      int ne = e, ns = s, nc = c;
      const bool more = advance(ne, ns, nc);
      const int ne1 = ne, ns1 = ns, nc1 = nc;  // the next chunk: gathered below, by the warps without a tile in the narrowest layer
      __pipeline_wait_prior(0);              // this chunk's rows (requested during the previous chunk) have landed
      __syncthreads();
      stamp(0);
      const bool more2 = more && advance(ne, ns, nc);  // (ne, ns, nc): the chunk after next
      const int pos0 = c * BR;                          // position of the chunk's first row in its mini-batch
      uint32_t drop_ks = 0u;                            // DROP: the key of optimizer step t_step
      if constexpr (DROP) {
        if (!val) {
          drop_ks = mix32(drop_key + (uint32_t)t_step * 0x9e3779b9U);
          if (a.drop_layers & 1u) {  // input dropout, in place on the staged rows (weight_step(0) reads them too)
            float* xs = smem + a.xofs[cur];
            const uint32_t thr = a.drop_thr[0];
            const float sc = a.drop_scale[0];
            for (int r = warp; r < nb; r += NWARPS) {  // live rows only: a padding row keeps its finite stale values
              const uint32_t kr = drop_row(drop_ks, pos0 + r, 0);
              for (int k = lane; k < n_in; k += 32) {
                const float v = xs[r * a.apitch[0] + k];
                xs[r * a.apitch[0] + k] = drop_keep(kr, k, thr) ? v * sc : 0.f;
              }
            }
            __syncthreads();
          }
        }
      }

      // ---- forward ---------------------------------------------------------------------------
      for (int l = 0; l < L; ++l) {
        const int Kp = a.im.kp[l], Np = a.im.np[l], N = a.net.dims[l + 1], act = a.net.act[l];
        const float* in = (l == 0) ? smem + a.xofs[cur] : smem + a.aofs[l];
        float* out = smem + a.aofs[l + 1];
        const int ip = a.apitch[l], op = a.apitch[l + 1];
        const float* Wl = sW + a.im.wofs[l];
        const float* bl = sW + a.im.bofs[l];
        const float l1c = a.net.l1[l] * (a.hp.l1_div_batch ? 1.f : (float)nbt);
        bool drop_out = false;  // DROP: this layer's activation is the input of a dropped layer
        uint32_t out_kr = 0u, out_thr = 0u;
        float out_sc = 1.f;
        if constexpr (DROP) {
          drop_out = !val && ((a.drop_layers >> (l + 1)) & 1u);
          if (drop_out) {
            out_kr = drop_row(drop_ks, pos0 + (lane & 7) + 8 * (lane >> 3), l + 1);  // the row this lane stores
            out_thr = a.drop_thr[l + 1];
            out_sc = a.drop_scale[l + 1];
          }
        }
        // cp.async of the next chunk: off the step's critical path (at the head of a chunk it cost 2 k cycles), half of the rows in each of
        // the two narrowest layers, by the warps without a tile there (a row costs its warp ~700 cycles of dependent address work)
        if (more && (l == a.gather_layer || l == a.gather_layer2)) {
          const int busy = min(Np >> 2, NWARPS), first = busy < NWARPS ? busy : 0;
          const bool both = a.gather_layer == a.gather_layer2, second = l == a.gather_layer;
          if (warp >= first) gather(cur ^ 1, ne1, ns1, nc1, first, NWARPS - first, (both || !second) ? 0 : BR / 2, (both || second) ? BR : BR / 2);
        }
        if (l == 0) {  // the last two warps have no tile in the first layer of a 64-tag hourglass (14 tiles): they prepare the next step
          if (warp == NWARPS - 1 && more2) stage_indices(cur, ne, ns, nc);  // read by the gather at the top of the next chunk
          if (warp == NWARPS - 2 && first_chunk && !val && lane == 0) {  // read after the loss barrier of step t+1
            if constexpr (OPT) s_opt[(t_step + 1) & 1] = gb::opt_step_next(a.opt, s_opt[t_step & 1]);
            else s_alpha[(t_step + 1) & 1] = adam_alpha(t_step + 1);
          }
        }
        // A warp owns 32 rows x 4 output columns; lane = (row group p, K quarter kq): rows p, p+8, p+16, p+24 against every fourth
        // block of four k.  Per block a lane loads 4 + 4 float4 for 64 FMA (a row per lane with the whole K needs 1 + 4 for 16: the
        // shared-memory return path, 128 B/clk, bounded these loops); the four K quarters are summed by a two-round reduce-scatter
        // over the lanes that leaves lane (p, kq) with row p + 8 kq.
        const int p8 = lane & 7, kq = lane >> 3, Kb = Kp >> 2;
        for (int task = warp; task < (Np >> 2); task += NWARPS) {
          const int n0 = task << 2;
          float acc[4][4];
#pragma unroll
          for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int c = 0; c < 4; ++c) acc[j][c] = 0.f;
          const float* arow = in + p8 * ip;
          const float* wcol = Wl + n0;
          for (int kb = kq; kb < Kb; kb += 4) {
            const int k = kb << 2;
            float4 av[4], wv[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) av[j] = *reinterpret_cast<const float4*>(arow + 8 * j * ip + k);
#pragma unroll
            for (int t = 0; t < 4; ++t) wv[t] = *reinterpret_cast<const float4*>(wcol + (k + t) * Np);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              acc[j][0] = fmaf(av[j].x, wv[0].x, acc[j][0]); acc[j][1] = fmaf(av[j].x, wv[0].y, acc[j][1]); acc[j][2] = fmaf(av[j].x, wv[0].z, acc[j][2]); acc[j][3] = fmaf(av[j].x, wv[0].w, acc[j][3]);
              acc[j][0] = fmaf(av[j].y, wv[1].x, acc[j][0]); acc[j][1] = fmaf(av[j].y, wv[1].y, acc[j][1]); acc[j][2] = fmaf(av[j].y, wv[1].z, acc[j][2]); acc[j][3] = fmaf(av[j].y, wv[1].w, acc[j][3]);
              acc[j][0] = fmaf(av[j].z, wv[2].x, acc[j][0]); acc[j][1] = fmaf(av[j].z, wv[2].y, acc[j][1]); acc[j][2] = fmaf(av[j].z, wv[2].z, acc[j][2]); acc[j][3] = fmaf(av[j].z, wv[2].w, acc[j][3]);
              acc[j][0] = fmaf(av[j].w, wv[3].x, acc[j][0]); acc[j][1] = fmaf(av[j].w, wv[3].y, acc[j][1]); acc[j][2] = fmaf(av[j].w, wv[3].z, acc[j][2]); acc[j][3] = fmaf(av[j].w, wv[3].w, acc[j][3]);
            }
          }
          float s4[4];
          quarter_reduce(acc, lane, s4);
          const int row = p8 + 8 * kq;
          const float4 bv = *reinterpret_cast<const float4*>(bl + n0);
          float4 o;
          o.x = (n0 + 0 < N) ? gb::apply_act(act, s4[0] + bv.x) : 0.f;
          o.y = (n0 + 1 < N) ? gb::apply_act(act, s4[1] + bv.y) : 0.f;
          o.z = (n0 + 2 < N) ? gb::apply_act(act, s4[2] + bv.z) : 0.f;
          o.w = (n0 + 3 < N) ? gb::apply_act(act, s4[3] + bv.w) : 0.f;
          if constexpr (DROP) {
            if (drop_out) {
              o.x = drop_keep(out_kr, n0 + 0, out_thr) ? o.x * out_sc : 0.f;
              o.y = drop_keep(out_kr, n0 + 1, out_thr) ? o.y * out_sc : 0.f;
              o.z = drop_keep(out_kr, n0 + 2, out_thr) ? o.z * out_sc : 0.f;
              o.w = drop_keep(out_kr, n0 + 3, out_thr) ? o.w * out_sc : 0.f;
            }
          }
          *reinterpret_cast<float4*>(out + row * op + n0) = o;
          if (l1c != 0.f && row < nb) acc_reg += l1c * (fabsf(o.x) + fabsf(o.y) + fabsf(o.z) + fabsf(o.w));
        }
        __syncthreads();
        stamp(1 + l);
      }

      // ---- loss, accuracy, dz of the output layer: dz = (dL/dyhat + l1*sign(a)) * act'(a) ---------------
      {
        const float* yh = smem + a.aofs[L];
        const int yp = a.apitch[L];
        const float* yt = smem + a.yofs[cur];
        float* G = dz_buf(0);
        const int NpL = a.im.np[L - 1], actL = a.net.act[L - 1];
        const float cL = a.net.l1[L - 1] / (a.hp.l1_div_batch ? (float)nbt : 1.f);
        const float gscale = 2.f / ((float)nbt * (float)n_out);
        const int loss = LOSS ? a.hp.loss : GB_LOSS_MSE;  // launch-uniform; MSE keeps its own arithmetic (d * d, gscale * d)
        const float lscale = 1.f / ((float)nbt * (float)n_out);
        for (int r = warp; r < BR; r += NWARPS) {
          // keras "accuracy" on 2-D float targets: argmax match (binary if width 1); first maximum wins, as np.argmax.  The
          // values are compared as order-preserving integer keys so that the warp-wide maximum is one REDUX.
          unsigned kp = 0u, kt = 0u;
          int bp = 0x7fffffff, bt = 0x7fffffff;
          for (int j = lane; j < NpL; j += 32) {
            float g = 0.f;
            if (r < nb && j < n_out) {
              const float ao = yh[r * yp + j], t = yt[r * a.ypitch + j];
              if (loss == GB_LOSS_MSE) {
                const float d = ao - t;
                // one fused multiply-add, pinned: in the LOSS kernels the compiler may otherwise merge the two branches' sums into
                // one add of a separately rounded d * d, and an MSE fit's loss there would differ in the last bits from the MSE kernels'
                acc_sq = __fmaf_rn(d, d, acc_sq);
                g = gscale * d;
              } else {
                acc_sq += gb::loss_value(loss, ao, t);
                g = lscale * gb::loss_grad(loss, ao, t);
              }
              if (cL != 0.f) g += cL * ((ao > 0.f) ? 1.f : ((ao < 0.f) ? -1.f : 0.f));
              g *= gb::act_grad_from_output(actL, ao);
              const unsigned ka = order_key(ao), kb = order_key(t);
              if (ka > kp) { kp = ka; bp = j; }
              if (kb > kt) { kt = kb; bt = j; }
              if (n_out == 1) acc_hit += ((ao > 0.5f ? 1.f : 0.f) == t) ? 1.f : 0.f;
            }
            G[r * a.dpitch + j] = g;
          }
          if (n_out > 1 && r < nb) {
            const unsigned mp = __reduce_max_sync(0xffffffffu, kp), mt = __reduce_max_sync(0xffffffffu, kt);
            const int ip = __reduce_min_sync(0xffffffffu, kp == mp ? bp : 0x7fffffff);
            const int it = __reduce_min_sync(0xffffffffu, kt == mt ? bt : 0x7fffffff);
            if (lane == 0) acc_hit += (ip == it) ? 1.f : 0.f;
          }
        }
      }
      __syncthreads();
      stamp(L + 1);
      const float alpha = OPT ? 0.f : s_alpha[t_step & 1];
      gb::OptStep ost{};
      if constexpr (OPT) ost = s_opt[t_step & 1];

      // ---- backward + Adam, pipelined over the layers ------------------------------------------------------
      // dz of layer l lives in D buffer (L-1-l) % 3.  Phase p (one barrier each) runs, on disjoint data,
      //   B(p):   dz_{p-1} = (dz_p . W_p^T + l1*sign(a)) * act'(a)      warps from the top, one 4-column task each
      //   C(p+1): dW = a_in^T . dz, db, Adam in place                    all threads, one 4x2 block of W each
      // B(p) reads W_p while C(p+1) writes W_{p+1}; the third buffer keeps dz_{p+1} alive while B(p) writes dz_{p-1}.
      auto input_grad = [&](int l) {  // B(l), l >= 1
        const int Kp = a.im.kp[l], Np = a.im.np[l], K = a.net.dims[l], actp = a.net.act[l - 1];
        const float* D = dz_buf((L - 1 - l) % 3);
        float* Dn = dz_buf((L - l) % 3);
        const float* Wl = sW + a.im.wofs[l];
        const float* aprev = smem + a.aofs[l];  // output of layer l-1
        const float cp = a.net.l1[l - 1] / (a.hp.l1_div_batch ? (float)nbt : 1.f);
        const int p8 = lane & 7, kq = lane >> 3, Nb = Np >> 2;  // lane = (row group, quarter of the n blocks): as in the forward pass
        bool drop_in = false;  // DROP: layer l's input was dropped in the forward pass
        uint32_t in_kr = 0u, in_thr = 0u;
        float in_sc = 1.f;
        if constexpr (DROP) {
          drop_in = (a.drop_layers >> l) & 1u;
          if (drop_in) {
            in_kr = drop_row(drop_ks, pos0 + p8 + 8 * kq, l);
            in_thr = a.drop_thr[l];
            in_sc = a.drop_scale[l];
          }
        }
        for (int task = NWARPS - 1 - warp; task < (Kp >> 2); task += NWARPS) {
          const int k0 = task << 2;
          float acc[4][4];
#pragma unroll
          for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int c = 0; c < 4; ++c) acc[j][c] = 0.f;
          const float* drow = D + p8 * a.dpitch;
          const float* wrow = Wl + k0 * Np;
          for (int nb4 = kq; nb4 < Nb; nb4 += 4) {
            const int nn = nb4 << 2;
            float4 dv[4], wv[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) dv[j] = *reinterpret_cast<const float4*>(drow + 8 * j * a.dpitch + nn);
#pragma unroll
            for (int c = 0; c < 4; ++c) wv[c] = *reinterpret_cast<const float4*>(wrow + c * Np + nn);
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
              for (int c = 0; c < 4; ++c) {
                acc[j][c] = fmaf(dv[j].x, wv[c].x, acc[j][c]);
                acc[j][c] = fmaf(dv[j].y, wv[c].y, acc[j][c]);
                acc[j][c] = fmaf(dv[j].z, wv[c].z, acc[j][c]);
                acc[j][c] = fmaf(dv[j].w, wv[c].w, acc[j][c]);
              }
          }
          float s4[4];
          quarter_reduce(acc, lane, s4);
          const int row = p8 + 8 * kq;
          const bool live = row < nb;
          const float4 ao = *reinterpret_cast<const float4*>(aprev + row * a.apitch[l] + k0);
          auto dz = [&](float g, float o, int j) -> float {
            if (!live || j >= K) return 0.f;
            if constexpr (DROP) {
              if (drop_in) {  // dropped: no gradient; kept: g s act'(a), a = stored value / s
                if (!drop_keep(in_kr, j, in_thr)) return 0.f;
                g *= in_sc;
                o = o / in_sc;
              }
            }
            if (cp != 0.f) g += cp * ((o > 0.f) ? 1.f : ((o < 0.f) ? -1.f : 0.f));
            return g * gb::act_grad_from_output(actp, o);
          };
          float4 o;
          o.x = dz(s4[0], ao.x, k0 + 0); o.y = dz(s4[1], ao.y, k0 + 1); o.z = dz(s4[2], ao.z, k0 + 2); o.w = dz(s4[3], ao.w, k0 + 3);
          *reinterpret_cast<float4*>(Dn + row * a.dpitch + k0) = o;
        }
      };
      float pen_next = 0.f;  // REG: this thread's share of the penalty of the weights this step writes
      auto weight_step = [&](int l) {  // C(l)
        const int Kp = a.im.kp[l], Np = a.im.np[l];
        const float* D = dz_buf((L - 1 - l) % 3);
        const float* ain = (l == 0) ? smem + a.xofs[cur] : smem + a.aofs[l];
        const int ip = a.apitch[l];
        float* Wl = sW + a.im.wofs[l];
        float* Ml = Mg + a.im.wofs[l];
        float* Vl = Vg + a.im.wofs[l];
        float* Gl = Gacc + a.im.wofs[l];
        const int nhalf = Np >> 1, nblocks = (Kp >> 2) * nhalf;
        for (int bid = tid; bid < nblocks; bid += THREADS) {  // consecutive threads along n: the moments stream coalesced
          const int kb = bid / nhalf, n0 = (bid - kb * nhalf) << 1, k0 = kb << 2;
          const bool adam = nchunks == 1 || last_chunk;
          float2 mq[4], vq[4];  // Adam moments of this block: requested now, consumed after the reduction over the batch rows
          if (adam) {
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              mq[i] = *reinterpret_cast<const float2*>(Ml + (k0 + i) * Np + n0);
              vq[i] = *reinterpret_cast<const float2*>(Vl + (k0 + i) * Np + n0);
            }
          }
          float2 gs[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) gs[i] = make_float2(0.f, 0.f);
#pragma unroll 4
          for (int r = 0; r < BR; ++r) {
            const float4 av = *reinterpret_cast<const float4*>(ain + r * ip + k0);
            const float2 d = *reinterpret_cast<const float2*>(D + r * a.dpitch + n0);
            gs[0].x = fmaf(av.x, d.x, gs[0].x); gs[0].y = fmaf(av.x, d.y, gs[0].y);
            gs[1].x = fmaf(av.y, d.x, gs[1].x); gs[1].y = fmaf(av.y, d.y, gs[1].y);
            gs[2].x = fmaf(av.z, d.x, gs[2].x); gs[2].y = fmaf(av.z, d.y, gs[2].y);
            gs[3].x = fmaf(av.w, d.x, gs[3].x); gs[3].y = fmaf(av.w, d.y, gs[3].y);
          }
          if (nchunks > 1) {  // multi-chunk mini-batch: sum the chunks' gradients in the L2 scratch image; Adam with the last chunk
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              float2* gp = reinterpret_cast<float2*>(Gl + (k0 + i) * Np + n0);
              if (!first_chunk) {
                const float2 o = *gp;
                gs[i].x += o.x; gs[i].y += o.y;
              }
              if (!last_chunk) *gp = gs[i];
            }
          }
          if (adam) {
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const int off = (k0 + i) * Np + n0;
              float2 w = *reinterpret_cast<float2*>(Wl + off);
              float2 m = mq[i];
              float2 v = vq[i];
              if constexpr (REG) {  // once per step, on the summed gradient, before clipvalue and the rule
                const float c1 = a.reg.kernel_l1[l], c2 = 2.f * a.reg.kernel_l2[l];
                gs[i].x += c1 * gb::sign0(w.x) + c2 * w.x;
                gs[i].y += c1 * gb::sign0(w.y) + c2 * w.y;
              }
              if constexpr (OPT) {  // m / v: the optimizer's state slots 0 / 1
                gb::opt_update(a.opt, ost, w.x, gs[i].x, m.x, v.x);
                gb::opt_update(a.opt, ost, w.y, gs[i].y, m.y, v.y);
              } else {
                adam_update(w.x, gs[i].x, m.x, v.x, alpha, omb1, omb2, eps);
                adam_update(w.y, gs[i].y, m.y, v.y, alpha, omb1, omb2, eps);
              }
              *reinterpret_cast<float2*>(Wl + off) = w;
              *reinterpret_cast<float2*>(Ml + off) = m;
              *reinterpret_cast<float2*>(Vl + off) = v;
              if constexpr (REG) {  // real entries only, never the padding of the [Kp][Np] image
                const int K = a.net.dims[l], N = a.net.dims[l + 1];
                const float c1 = a.reg.kernel_l1[l], c2 = a.reg.kernel_l2[l];
                if (k0 + i < K && n0 < N) pen_next += c1 * fabsf(w.x) + c2 * (w.x * w.x);
                if (k0 + i < K && n0 + 1 < N) pen_next += c1 * fabsf(w.y) + c2 * (w.y * w.y);
              }
            }
          }
        }
        for (int j = THREADS - 1 - tid; j < Np; j += THREADS) {
          float g = 0.f;
          for (int r = 0; r < BR; ++r) g += D[r * a.dpitch + j];
          const int off = a.im.bofs[l] + j;
          if (nchunks > 1) {
            if (!first_chunk) g += Gacc[off];
            if (!last_chunk) { Gacc[off] = g; continue; }
          }
          float w = sW[off], m = Mg[off], v = Vg[off];
          if constexpr (REG) g += a.reg.bias_l1[l] * gb::sign0(w) + 2.f * a.reg.bias_l2[l] * w;
          if constexpr (OPT) gb::opt_update(a.opt, ost, w, g, m, v);
          else adam_update(w, g, m, v, alpha, omb1, omb2, eps);
          sW[off] = w; Mg[off] = m; Vg[off] = v;
          if constexpr (REG)
            if (j < a.net.dims[l + 1]) pen_next += a.reg.bias_l1[l] * fabsf(w) + a.reg.bias_l2[l] * (w * w);
        }
      };
      if (!val) {
        for (int p = L - 1; p >= 0; --p) {
          if (p > 0) input_grad(p);
          if (p + 1 < L) weight_step(p + 1);
          if (p == 0) weight_step(0);
          __syncthreads();
          stamp(L + 2 + (L - 1 - p));
        }
        if constexpr (REG)
          if (last_chunk) pen = pen_next;  // the optimizer step ran: the next forward pass uses the weights it wrote
      }
      cur ^= 1;
     }  // chunks
    }
    if (vsteps > 0) epoch_stats(acc_sq, acc_reg, acc_hit, a.out_val_loss, a.out_val_acc, nv, e);
    else epoch_stats(acc_sq, acc_reg, acc_hit, a.out_loss, a.out_acc, n, e);
    if (stopping) {
      // the history entries of epoch e are written (by thread 0, after the last barrier of epoch_stats): apply the rule to the
      // monitored one, widened to double as Python compares it.  Bit 0 of the decision: snapshot; bit 1: stop.
      if (tid == 0) {
        const gb_fit_stop rule = a.stop[job_id];
        const float* monitored = rule.monitor == 0 ? a.out_loss : rule.monitor == 1 ? a.out_acc
                               : vsteps == 0 ? nullptr : rule.monitor == 2 ? a.out_val_loss : rule.monitor == 3 ? a.out_val_acc : nullptr;
        auto improves = [&](double v, double ref) -> bool {
          return rule.mode > 0 ? v + rule.min_delta < ref : v - rule.min_delta > ref;
        };
        int act = 0;
        if (monitored != nullptr && e >= rule.start_from_epoch) {
          const float v = monitored[(long)job_id * a.hp.epochs + e];
          if (rule.restore_best && best_epoch < 0) { act |= 1; best_epoch = e; }
          ++wait;
          if (improves(v, best)) {
            best = v;
            best_epoch = e;
            if (rule.restore_best) act |= 1;
            if (!rule.has_baseline || improves(v, rule.baseline)) wait = 0;
          } else if (wait >= rule.patience && e > 0) {
            act |= 2;
          }
        }
        if (act & 2) { a.out_epochs[job_id] = e + 1; }
        reinterpret_cast<volatile int*>(s_red[0])[0] = act;
      }
      __syncthreads();
      const int act = reinterpret_cast<volatile int*>(s_red[0])[0];
      if (act & 1) write_image(a.best_params + (long)job.slot * a.pstride);
      if (act & 2) {
        __pipeline_wait_prior(0);  // the next epoch's first chunk is in flight
        break;
      }
    }
  }

  // ---- trained weights (or, with restore_best, the snapshot) back to the canonical layout ------------------------------
  if (stopping) {
    bool restore = false;
    if (tid == 0) {
      restore = a.stop[job_id].restore_best && best_epoch >= 0;
      a.out_best_epoch[job_id] = best_epoch;
    }
    if (__syncthreads_or(restore)) {  // the snapshot's threads are not this copy's
      const float* B = a.best_params + (long)job.slot * a.pstride;
      const int count = a.im.pofs[L - 1] + a.net.dims[L - 1] * a.net.dims[L] + a.net.dims[L];
      for (int i = tid; i < count; i += THREADS) P[i] = B[i];
    } else {
      write_image(P);
    }
  } else {
    write_image(P);
  }
  if (tracing) {
    stamp(2 * L + 3);  // epoch statistics + write-back
    for (int i = 0; i < 2 * GB_MAX_LAYERS + 4; ++i) a.trace[i] = s_phase[i];
  }
