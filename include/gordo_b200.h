/*
 * gordo_b200.h -- C ABI of the H100 (sm_90a) implementation of gordo's per-machine
 * autoencoder train-and-score hot path.
 *
 * The reference (equinor/gordo-components) has no native FFI: its plug-in boundary is a
 * Python class path + the sklearn/GordoBase protocol (gordo/machine/model/base.py:10-35,
 * gordo/machine/model/anomaly/base.py:11-23, gordo/serializer/from_definition.py:176-191).
 * This header is the seam *below* that protocol: every arithmetic library call the
 * reference makes on the hot path (Keras Model.predict / Model.fit, sklearn MinMaxScaler,
 * pandas rolling/abs/mean in DiffBasedAnomalyDetector) maps to one entry point here.
 * Each entry point cites the reference call it replaces.  INTEGRATION.md shows the
 * ctypes binding (gordo_components_b200/_cabi.py is the live copy).
 *
 * Conventions
 *  - plain C: pointers and sizes only, no torch types.  Unless stated otherwise every
 *    pointer is a DEVICE pointer owned by the caller; nothing here allocates or frees.
 *  - every function enqueues on `stream` (a cudaStream_t passed as void*) and returns
 *    without synchronising.  Return value: 0 or a negative gb_status; the message of
 *    the last failure on the calling thread is available from gb_last_error().
 *  - float32 everywhere on device; row-major; rows of all machines are concatenated:
 *    x[total_rows][n_features], y / outputs [total_rows][n_features_out].
 *  - a *slot* is one trained network (a machine, or one CV fold of a machine); a *job*
 *    binds a slot to a contiguous range of rows.
 */
#ifndef GORDO_B200_H
#define GORDO_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GB_ABI_VERSION 2
#define GB_MAX_LAYERS 16
#define GB_MAX_WIDTH 256 /* widest layer / feature count (the feedforward_model / feedforward_symmetric defaults are 256-128-64) */

typedef enum gb_status {
  GB_OK = 0,
  GB_E_ARG = -1,     /* null pointer / bad enum / inconsistent sizes          -> ValueError  */
  GB_E_SHAPE = -2,   /* architecture outside what the kernels support          -> ValueError  */
  GB_E_ALIGN = -3,   /* pointer not 16-byte aligned                            -> ValueError  */
  GB_E_SMEM = -4,    /* architecture does not fit in shared memory             -> ValueError  */
  GB_E_CUDA = -5,    /* CUDA runtime error (message has cudaGetErrorString)    -> RuntimeError*/
  GB_E_DEVICE = -6   /* no sm_90 device                                        -> RuntimeError*/
} gb_status;

typedef enum gb_act { GB_ACT_LINEAR = 0, GB_ACT_TANH = 1, GB_ACT_RELU = 2, GB_ACT_SIGMOID = 3 } gb_act;

/* Training loss (the `loss` of the reference's compile_kwargs, a Keras 3 loss name).  With e = yhat - y and eps = 1e-7, each is a
 * per-element f averaged over all B * n_out elements of a mini-batch (Keras' per-sample mean, then sum_over_batch_size):
 *   MSE e^2;  MAE |e|;  MAPE 100 |e| / max(|y|, eps);  MSLE (log(max(yhat, eps) + 1) - log(max(y, eps) + 1))^2;
 *   HUBER 0.5 e^2 if |e| <= 1 else |e| - 0.5 (delta 1);  LOG_COSH e + softplus(-2 e) - log 2.
 * Gradients follow TF: sign(0) = 0 for MAE / MAPE, and MSLE passes none where yhat < eps. */
typedef enum gb_loss {
  GB_LOSS_MSE = 0,
  GB_LOSS_MAE = 1,
  GB_LOSS_MAPE = 2,
  GB_LOSS_MSLE = 3,
  GB_LOSS_HUBER = 4,
  GB_LOSS_LOG_COSH = 5
} gb_loss;

/* Dense stack built by feedforward_model / feedforward_symmetric / feedforward_hourglass
 * (gordo/machine/model/factories/feedforward_autoencoder.py:65-104).  dims[0] = n_features,
 * dims[l+1] = units of Dense layer l; l1[l] = activity_regularizer l1 coefficient of layer l
 * (10e-5 on encoder layers i>=1, :80-81), used by training only. */
typedef struct gb_ffnet {
  int32_t n_layers;
  int32_t dims[GB_MAX_LAYERS + 1];
  int32_t act[GB_MAX_LAYERS];
  float l1[GB_MAX_LAYERS];
} gb_ffnet;

/* One unit of work: network `slot` applied to rows [x_row, x_row + n_rows) of x / y,
 * results written to rows [out_row, out_row + n_rows) of the output arrays. */
typedef struct gb_job {
  int32_t slot;
  int32_t n_rows;
  int64_t x_row;
  int64_t out_row;
} gb_job;

/* ---- library ------------------------------------------------------------------------ */
int gb_abi_version(void);
const char* gb_last_error(void);
/* 0 if `device` is an sm_90 (H100) part; GB_E_DEVICE otherwise.  Fills sm count if non-null. */
int gb_device_check(int device, int* sm_count);

/* ---- parameter layout ---------------------------------------------------------------
 * Canonical per-slot parameter vector ("Keras order"): for each layer l: kernel
 * W_l[dims[l]][dims[l+1]] row-major (Keras Dense kernel layout [in,out]) then bias
 * b_l[dims[l+1]].  Slots are `gb_ffnet_param_stride()` floats apart (count rounded up to 4). */
size_t gb_ffnet_param_count(const gb_ffnet* net);
size_t gb_ffnet_param_stride(const gb_ffnet* net);

/* ---- K1+K4: predict + anomaly score, fused --------------------------------------------
 * Replaces, per job: KerasBaseEstimator.predict -> keras Model.predict
 * (gordo/machine/model/models.py:289-300) and the arithmetic of
 * DiffBasedAnomalyDetector.anomaly (gordo/machine/model/anomaly/diff.py:350-385, 420-444):
 *   out_model            = net(x)                                   [rows][n_out]
 *   out_tag_unscaled     = |out_model - y|                          [rows][n_out]
 *   out_tag_scaled       = |out_model - y| * scale[slot]            [rows][n_out]   (MinMax offset cancels)
 *   out_total_unscaled   = mean_j(out_tag_unscaled^2)               [rows]
 *   out_total_scaled     = mean_j(out_tag_scaled^2)                 [rows]
 *   out_conf             = out_tag_unscaled / feat_thr[slot]        [rows][n_out]   (diff.py:421 uses the unscaled diff)
 *   out_total_conf       = out_total_scaled / agg_thr[slot]         [rows]
 * y == NULL -> prediction only (all score outputs must be NULL).  Any score output may be
 * NULL and is then skipped; feat_thr / agg_thr NULL -> the confidences must be NULL.
 * params: [n_slots][param_stride]; scale, feat_thr: [n_slots][n_out]; agg_thr: [n_slots].
 * jobs: DEVICE array of n_jobs gb_job; max_rows = max n_rows over jobs (host value, sizes the grid).
 * n_x_rows / n_out_rows: number of rows of the x (and y) array and of the output arrays (TMA tensor extents).
 * variant (low byte): 0 = auto (tensor-core kernel for the stacks it covers, the row-per-thread kernel for stacks whose widths are
 * all <= 16, else the generic one), 1 = generic fp32 CUDA-core kernel, 2 = tensor-core (wgmma) split-precision kernel, 3 = row-per-thread
 * fp32 kernel (2 / 3: GB_E_SHAPE if the architecture is outside their range); higher bytes are debug knobs and must be 0.
 * Non-finite inputs stay in their own row.  The totals are the plain mean over all n_out tags (the numpy mean that threshold
 * fitting uses, diff.py:292): a NaN tag gives a NaN total and an infinite tag an infinite one.  pandas' skip-NaN mean of the
 * anomaly frame (diff.py:366, :383) is the caller's to apply.  NaN in x gives an all-NaN row.  On variants 1 and 3, ±inf in x
 * propagates as IEEE arithmetic does (tanh(±inf) = ±1, as in Keras).  Variant 2 splits x into a TF32 part and a BF16 remainder,
 * which is inf - inf = NaN, so ±inf in x gives an all-NaN row there: launch variant 1 for such rows. */
int gb_ffae_infer_score(const gb_ffnet* net, const float* params, const gb_job* jobs, int32_t n_jobs,
                        int32_t max_rows, int64_t n_x_rows, int64_t n_out_rows, const float* x, const float* y, const float* scale,
                        const float* feat_thr, const float* agg_thr, float* out_model,
                        float* out_tag_scaled, float* out_tag_unscaled, float* out_total_scaled,
                        float* out_total_unscaled, float* out_conf, float* out_total_conf,
                        int32_t variant, void* stream);

/* GB_OK if the tensor-core (variant 2) kernel covers this architecture, else GB_E_SHAPE. */
int gb_ffae_tc_supported(const gb_ffnet* net);

/* The launch plan of the generic (variant 1) kernel for this architecture, without launching: rows per tile (128, 64 or 32)
 * and whether every layer's weights stay resident in shared memory (1) or are staged layer by layer (0; a layer too large to
 * stage whole next to the activations is staged in blocks of output columns).  GB_E_SMEM exactly when gb_ffae_infer_score
 * would refuse the architecture on variant 1 for shared memory; either output may be NULL. */
int gb_ffae_infer_plan(const gb_ffnet* net, int32_t* rows_per_tile, int32_t* resident);

/* gb_ffae_infer_score behind a Pipeline's per-feature input scalers (sklearn MinMaxScaler / StandardScaler / RobustScaler /
 * MaxAbsScaler .transform in front of the network, composed into one affine map): x is float64 [n_x_rows][n_in], and the kernel
 * applies x' = (float)((x * x_scale[slot][c]) + x_offset[slot][c]) as it loads each element -- two roundings in double, no fma,
 * one rounding to float, exactly what gb_affine_f64 writes.  x_scale, x_offset: [n_slots][n_in] double, both non-NULL (GB_E_ARG).
 * Everything else -- arguments, variants, outputs, the handling of NaN and ±inf in x' -- is that of gb_ffae_infer_score, and the
 * result is bit for bit gb_affine_f64 followed by gb_ffae_infer_score with the same variant on the same device.  It reads x once
 * instead of reading it, writing x' and reading x' back.  Variant 2 stages twice the bytes per x tile: a stack whose weights
 * leave no room for them is GB_E_SMEM (see gb_ffae_infer_plan_x64), never a silent change of kernel. */
int gb_ffae_infer_score_x64(const gb_ffnet* net, const float* params, const gb_job* jobs, int32_t n_jobs, int32_t max_rows,
                            int64_t n_x_rows, int64_t n_out_rows, const double* x, const double* x_scale, const double* x_offset,
                            const float* y, const float* scale, const float* feat_thr, const float* agg_thr, float* out_model,
                            float* out_tag_scaled, float* out_tag_unscaled, float* out_total_scaled, float* out_total_unscaled,
                            float* out_conf, float* out_total_conf, int32_t variant, void* stream);

/* The kernel gb_ffae_infer_score_x64 runs for this architecture and variant (0..3, no debug bits), without launching and without
 * a device: *kernel = 1, 2 or 3 (0 resolved as gb_ffae_infer_score resolves it), *tc_warpgroups = warpgroups per CTA of the
 * tensor-core launch (3, or 2 when three warpgroups' float64 x tiles do not fit next to the weights; 0 for kernels 1 and 3).
 * GB_E_SHAPE / GB_E_SMEM exactly when gb_ffae_infer_score_x64 refuses the architecture on that variant; either output may be NULL. */
int gb_ffae_infer_plan_x64(const gb_ffnet* net, int32_t variant, int32_t* kernel, int32_t* tc_warpgroups);

/* ---- K4 alone: anomaly score of predictions that already exist ----------------------------
 * Same outputs as gb_ffae_infer_score, for a `yhat` produced elsewhere (a base estimator that is not
 * one of ours, e.g. the sklearn regressors the reference's detector tests use; an LSTM prediction from
 * gb_lstm_infer).  yhat and all outputs are indexed by out_row, y by x_row.  A NaN or ±inf in yhat or y reaches only
 * its own (row, tag) cells and that row's totals, which are the plain mean over all tags as in gb_ffae_infer_score. */
int gb_anomaly_score(const gb_job* jobs, int32_t n_jobs, int32_t max_rows, const float* yhat, const float* y,
                     int32_t n_out, const float* scale, const float* feat_thr, const float* agg_thr,
                     float* out_tag_scaled, float* out_tag_unscaled, float* out_total_scaled,
                     float* out_total_unscaled, float* out_conf, float* out_total_conf, void* stream);

/* The same arithmetic in float64, as the reference does it (pandas on float64 y: diff.py:268-300 `_scaled_mse_per_timestep`,
 * `_absolute_error`; :350-385, 420-444 in `anomaly`) -- used whenever the predictions did not come out of one of this
 * package's fp32 networks fused with the scoring (foreign base estimators, LSTM outputs): at data magnitude ~100 a float32
 * |yhat - y| is uncertain by 7.6e-6, i.e. percents of a small residual.  All arrays double. */
int gb_anomaly_score_f64(const gb_job* jobs, int32_t n_jobs, int32_t max_rows, const double* yhat, const double* y,
                         int32_t n_out, const double* scale, const double* feat_thr, const double* agg_thr,
                         double* out_tag_scaled, double* out_tag_unscaled, double* out_total_scaled,
                         double* out_total_unscaled, double* out_conf, double* out_total_conf, void* stream);

/* A TransformedTargetRegressor(transformer=MinMaxScaler) prediction, inverse-transformed and scored in float64 in one pass: for
 * every element, v = (float)((double)(float)((double)p - y_min) / y_scale) (sklearn's MinMaxScaler.inverse_transform on the float32
 * prediction, as gb_minmax_inverse_f32) goes to out_model, and (double)v is scored against y exactly as gb_anomaly_score_f64 scores
 * it, in the same order.  Every output is bit for bit gb_minmax_inverse_f32 followed by gb_anomaly_score_f64 on the widened
 * result, without the float64 copy of the prediction in between.  p (the network's raw float32 output), out_model and the score
 * outputs are indexed by out_row, y by x_row; p and out_model may be the same array.  y_scale / y_min: [n_slots][n_out], the
 * transformer's scale_ / min_.  scale / feat_thr / agg_thr and every score output as gb_anomaly_score_f64 (any output may be NULL). */
int gb_minmax_inverse_score_f64(const gb_job* jobs, int32_t n_jobs, int32_t max_rows, const float* p, const double* y,
                                int32_t n_out, const double* y_scale, const double* y_min, const double* scale,
                                const double* feat_thr, const double* agg_thr, float* out_model,
                                double* out_tag_scaled, double* out_tag_unscaled, double* out_total_scaled,
                                double* out_total_unscaled, double* out_conf, double* out_total_conf, void* stream);

/* ---- K7: MinMaxScaler.fit on the targets (diff.py:173; sklearn MinMaxScaler [3P]) -------
 * per job: scale[slot][j] = 1/(max_j - min_j) (zero range -> 1), offset[slot][j] = -min_j*scale.
 * minmax_ws: workspace [n_slots][2][n_out] floats (overwritten). */
int gb_minmax_fit(const gb_job* jobs, int32_t n_jobs, int32_t max_rows, const float* y, int32_t n_out,
                  float* scale, float* offset, float* minmax_ws, int32_t n_slots, void* stream);

/* Column extrema of float64 targets, for the scaler of a single detector (`scaler.fit(y)` sees float64 y in the reference):
 * minmax[slot][0][j] = min, minmax[slot][1][j] = max over the job's rows (NaNs skipped; +inf / -inf when there is no finite
 * sample).  sklearn's float64 scale_ / min_ arithmetic on them stays on the host. */
int gb_minmax_f64(const gb_job* jobs, int32_t n_jobs, int32_t max_rows, const double* y, int32_t n_out, double* minmax,
                  int32_t n_slots, void* stream);

/* ---- K5: thresholds of one CV fold (diff.py:222-233) ------------------------------------
 *   feat_thr[slot][j] = max_t min(tag_unscaled[t-window+1 .. t][j])   (rolling(window).min().max())
 *   agg_thr[slot]     = max_t min(total_scaled[t-window+1 .. t])
 * rows are taken at [out_row, out_row+n_rows) of the score arrays produced by
 * gb_ffae_infer_score for the fold's test rows.  n_rows < window -> NaN (pandas semantics). */
int gb_thresholds(const gb_job* jobs, int32_t n_jobs, int32_t max_rows, const float* tag_unscaled,
                  const float* total_scaled, int32_t n_out, int32_t window, float* feat_thr,
                  float* agg_thr, int32_t n_slots, void* stream);

/* float64 form for the score arrays of gb_anomaly_score_f64 (min / max select, so the thresholds are exact). */
int gb_thresholds_f64(const gb_job* jobs, int32_t n_jobs, int32_t max_rows, const double* tag_unscaled,
                      const double* total_scaled, int32_t n_out, int32_t window, double* feat_thr,
                      double* agg_thr, int32_t n_slots, void* stream);

/* Both fold thresholds of a detector with a smoothing window in one pass over the score arrays: feat_thr0 / agg_thr0 are
 * gb_thresholds at window w0 (the 6-row thresholds), feat_thr1 / agg_thr1 at window w1 (the smooth ones), bit for bit.  The
 * rolling minimum costs the same per row whatever the windows (van Herk / Gil-Werman blocks).  tag_unscaled, feat_thr0 and
 * feat_thr1 are all NULL or all set, and so are total_scaled, agg_thr0 and agg_thr1.  n_out in [1, GB_MAX_WIDTH], w0, w1 >= 1,
 * max_rows, n_jobs, n_slots >= 0; any other value is GB_E_ARG / GB_E_SHAPE naming the field, before any launch.  When a warp's
 * w0 + w1 buffer values do not fit in shared memory, the launch allocates a scratch area of at most 64 MB on the stream. */
int gb_thresholds_pair(const gb_job* jobs, int32_t n_jobs, int32_t max_rows, const float* tag_unscaled,
                       const float* total_scaled, int32_t n_out, int32_t w0, int32_t w1, float* feat_thr0,
                       float* agg_thr0, float* feat_thr1, float* agg_thr1, int32_t n_slots, void* stream);
int gb_thresholds_pair_f64(const gb_job* jobs, int32_t n_jobs, int32_t max_rows, const double* tag_unscaled,
                           const double* total_scaled, int32_t n_out, int32_t w0, int32_t w1, double* feat_thr0,
                           double* agg_thr0, double* feat_thr1, double* agg_thr1, int32_t n_slots, void* stream);

/* ---- K8: column moments behind the builder's cross-validation metrics (build_model.py:250-289, 378-446) ----
 * For job i, over rows yhat[out_row .. out_row+n_rows) and y[x_row .. x_row+n_rows), with e = yhat - y and
 * y0 = the job's first target row:  out[i][q][j] (double) = q0: sum e, q1: sum e^2, q2: sum |e|,
 * q3: sum (y - y0), q4: sum (y - y0)^2.  explained_variance / r2 / mean_squared_error / mean_absolute_error
 * (per tag and uniform-averaged, under any per-tag affine scoring scaler) follow from these on the host. */
int gb_cv_moments(const gb_job* jobs, int32_t n_jobs, const float* yhat, const float* y, int32_t n_out,
                  double* out, void* stream);

/* ---- K6: optional smoothing of anomaly columns (diff.py:302-308, 387-415) ------------------
 * method 0 = smm rolling(window).median(), 1 = sma rolling(window).mean() (first window-1 rows NaN; a window holding a NaN
 * gives NaN), 2 = ewma ewm(span=window).mean() (adjust=True, ignore_na=False: a NaN adds no observation, ages the weights and the
 * previous average is carried forward).  arr / out: [rows][n_cols], rows taken at [out_row, out_row+n_rows); max_rows = max n_rows
 * over jobs (sizes the row-chunk grid of the rolling kernels).  The rolling median keeps one sorted window per thread in shared
 * memory: windows up to 51 200 rows. */
int gb_smooth(const gb_job* jobs, int32_t n_jobs, int32_t max_rows, const float* arr, int32_t n_cols, int32_t window, int32_t method,
              float* out, void* stream);

/* The four smoothed anomaly arrays of a ragged batch of requests in one launch (one per 65 535 jobs): tag_scaled / tag_unscaled
 * [rows][n_tags] and total_scaled / total_unscaled [rows], float32 (in_f64 = 0) or float64 (in_f64 = 1, each value rounded to
 * float32 as it is read).  Job i smooths rows [out_row, out_row+n_rows) of each array into the same rows of the float32 output of
 * the same shape; its windows start at its own first row.  method / window as gb_smooth, the same for every job.  Every column
 * comes out bit for bit what gb_smooth gives for that array (as float32) alone: both run the same per-column code. */
int gb_smooth_scores(const gb_job* jobs, int32_t n_jobs, int32_t max_rows, const void* tag_scaled, const void* total_scaled,
                     const void* tag_unscaled, const void* total_unscaled, int32_t in_f64, int32_t n_tags, int32_t window, int32_t method,
                     float* smooth_tag_scaled, float* smooth_total_scaled, float* smooth_tag_unscaled, float* smooth_total_unscaled,
                     void* stream);

/* ---- K9: percentile thresholds of DiffBasedKFCVAnomalyDetector (diff.py:623-635: smoothed validation metric
 * .quantile(threshold_percentile)).  out[job][c] = q-quantile (linear interpolation, NaNs skipped -- pandas
 * semantics) of column c of rows [out_row, out_row+n_rows) of arr [rows][n_cols].  Jobs of up to 32768 rows are sorted in shared
 * memory; longer ones (a year of 10-minute data is ~52k rows) find the two order statistics by radix selection over L2. */
int gb_quantile(const gb_job* jobs, int32_t n_jobs, int32_t max_rows, const float* arr, int32_t n_cols, float q,
                float* out, void* stream);

/* ---- K8: per-feature affine pre-transform (sklearn MinMaxScaler/StandardScaler/... .transform in front of the
 * network inside a Pipeline: gordo serializer pipelines, e.g. examples/config_crd.yaml "sklearn.preprocessing.MinMaxScaler")
 *   out[out_row+r][c] = (float)(x[x_row+r][c] * a[slot][c] + b[slot][c]), computed in double like sklearn and rounded once,
 * i.e. exactly the float32 batch Keras sees.  (Folding a/b into the first Dense layer instead would cancel catastrophically
 * in fp32 for offset-dominated tags, so the transform stays a separate f64 pass.) */
int gb_affine_f64(const gb_job* jobs, int32_t n_jobs, int32_t max_rows, const double* x, int32_t n_cols, const double* a,
                  const double* b, float* out, void* stream);

/* ---- row permutations of the batched K-fold build (DiffBasedKFCVAnomalyDetector.cross_validate, diff.py:566-635) ----
 * Per job: dst row out_row + p = src row x_row + row_map[p] for p < n_rows; one map shared by every job (a KFold split is the
 * same for every machine of a bucket).  src / dst: [rows][n_cols] of elem_bytes (4 or 8) each; to_f32 = 1 reads float64 and
 * writes float32 (round to nearest), in the same pass.  Rows that are whole 16-byte units are copied 16 bytes at a time. */
int gb_gather_rows(const gb_job* jobs, int32_t n_jobs, int32_t max_rows, const int32_t* row_map, const void* src, int32_t n_cols,
                   int32_t elem_bytes, int32_t to_f32, void* dst, void* stream);

/* gb_gather_rows with a map per job, for buckets whose machines differ in length (each length has its own KFold split):
 * dst row out_row + p = src row x_row + row_map[map_ofs[i] + p] for job i and p < n_rows.  map_ofs: DEVICE array [n_jobs] of
 * offsets into row_map; jobs may share a map.  Element sizes, to_f32, the 16-byte path and the launches per 65 535 jobs as
 * gb_gather_rows; the same argument checks, and map_ofs must be non-NULL (GB_E_ARG), all before any launch. */
int gb_gather_rows_ragged(const gb_job* jobs, int32_t n_jobs, int32_t max_rows, const int32_t* row_map, const int64_t* map_ofs,
                          const void* src, int32_t n_cols, int32_t elem_bytes, int32_t to_f32, void* dst, void* stream);

/* MinMaxScaler.inverse_transform of float32 predictions, as sklearn does it inside TransformedTargetRegressor.predict: the
 * array stays float32 and each in-place step rounds to it, t = (float)((double)p - min_), v = (float)((double)t / scale_).
 * p indexed by x_row, outputs by out_row; scale / min_: [n_slots][n_cols] double.  out_f32 gets v, out_f64 gets (double)v;
 * either may be NULL, not both. */
int gb_minmax_inverse_f32(const gb_job* jobs, int32_t n_jobs, int32_t max_rows, const float* p, int32_t n_cols, const double* scale,
                          const double* min_, float* out_f32, double* out_f64, void* stream);

/* ---- K2: fit ---------------------------------------------------------------------------
 * Replaces scikeras KerasRegressor.fit -> keras Model.fit (models.py:284) for the Dense
 * stacks above: per job, `epochs` passes over rows [x_row, x_row+n_rows) in batches of
 * `batch_size`, loss = mean(f(net(x), y)) + sum_l l1[l]*sum|a_l| with f the gb_loss of hp->loss (mean squared error by
 * default), Adam (Keras defaults).  The history and the held-out statistics report the same loss.
 * One CTA per job trains the whole fit with weights resident in shared memory. */
typedef struct gb_fit_hparams {
  int32_t epochs;
  int32_t batch_size;
  int32_t shuffle;        /* 0: sequential order; 1: on-device keyed permutation per (seed, slot, epoch);
                             2: explicit `perm` (parity testing / reproducing a given order) */
  int32_t l1_div_batch;   /* 0: keras 3.3.3 behaviour (activity loss not divided by batch size) */
  float lr, beta1, beta2, eps;
  uint64_t seed;
  int32_t step0;          /* Adam step count already taken (warm start); 0 for a fresh fit */
  int32_t loss;           /* gb_loss; 0 = GB_LOSS_MSE.  Outside 0..5: GB_E_ARG, nothing enqueued */
} gb_fit_hparams;

/* Optimizer of a fit (the reference factories' `optimizer` / `optimizer_kwargs`, a Keras 3 optimizer; keras 3.3.3 update rules [3P],
 * restated, not verified against TF).  g is the summed mini-batch gradient of one parameter, t the 1-based step count of its slot
 * (hp->step0 / adam_t carry it across launches; the LSTM primer step counts), s0 / s1 the two state slots (adam_m / adam_v):
 *   ADAM, ADAMW  s0 = m += (g - m)(1 - beta1); s1 = v += (g^2 - v)(1 - beta2); w -= lr sqrt(1 - beta2^t) / (1 - beta1^t) m / (sqrt(v) + eps)
 *   RMSPROP      (rho = beta1) s0 = v = rho v + (1 - rho) g^2; d = v + eps, or with GB_OPT_CENTERED s1 = gbar = rho gbar + (1 - rho) g
 *                and d = v - gbar^2 + eps; inc = lr g / sqrt(d); with momentum > 0, s1 = mom = momentum mom + inc and w -= mom,
 *                else w -= inc.  Centered together with momentum would need a third slot: GB_E_ARG.
 *   ADAGRAD      s0 = acc += g^2 (at t = 1 the stored s0 is not read: acc starts from initial_accumulator); w -= lr g / sqrt(acc + eps)
 *   ADADELTA     (rho = beta1) s0 = Eg2 = rho Eg2 + (1 - rho) g^2; D = -sqrt(s1 + eps) g / sqrt(Eg2 + eps);
 *                s1 = rho s1 + (1 - rho) D^2; w += lr D
 *   ADAMAX       s0 = m += (g - m)(1 - beta1); s1 = u = max(beta2 u, |g|); w -= lr m / ((1 - beta1^t)(u + eps))
 *   NADAM        u_t = beta1 (1 - 0.96^t / 2), P_t = P_(t-1) u_t (float32 product from P_0 = 1, recomputed from step 1 by every launch);
 *                m, v as Adam; mhat = u_(t+1) m / (1 - P_t u_(t+1)) + (1 - u_t) g / (1 - P_t); w -= lr mhat / (sqrt(v / (1 - beta2^t)) + eps)
 * Before the update, every optimizer: g = clip(g, -clipvalue, clipvalue) when clipvalue > 0, then w -= w * weight_decay * lr.
 * Invalid (GB_E_ARG, nothing enqueued): an unknown kind or flag, a negative or non-finite lr, eps, momentum, initial_accumulator,
 * weight_decay or clipvalue, beta1 / beta2 (the ones the kind reads) outside [0, 1), GB_OPT_CENTERED on another kind than RMSPROP. */
typedef enum gb_opt {
  GB_OPT_ADAM = 0,
  GB_OPT_ADAMW = 1,
  GB_OPT_RMSPROP = 2,
  GB_OPT_ADAGRAD = 3,
  GB_OPT_ADADELTA = 4,
  GB_OPT_ADAMAX = 5,
  GB_OPT_NADAM = 6
} gb_opt;
#define GB_OPT_CENTERED 1 /* gb_optimizer.flags: RMSprop(centered=True) */

typedef struct gb_optimizer {
  int32_t kind;               /* gb_opt */
  int32_t flags;              /* GB_OPT_CENTERED or 0 */
  float lr;
  float beta1;                /* beta_1; rho of RMSPROP and ADADELTA */
  float beta2;                /* beta_2 of ADAM, ADAMW, ADAMAX, NADAM */
  float eps;
  float momentum;             /* RMSPROP */
  float initial_accumulator;  /* ADAGRAD */
  float weight_decay;         /* 0 = none */
  float clipvalue;            /* 0 = none */
} gb_optimizer;

/* The optimizer state (adam_m = slot 0, adam_v = slot 1) is opaque, in the kernel's padded layout: gb_ffae_fit_state_stride() floats
 * per slot; all zero for a fresh fit whatever the optimizer. */
size_t gb_ffae_fit_state_stride(const gb_ffnet* net);

/* params: [n_slots][param_stride], updated in place.  adam_m / adam_v: [n_slots][state_stride], updated in place
 * (all zero for a fresh fit).  Mini-batches above 32 rows are processed as 32-row chunks whose gradients are summed
 * before the optimizer step (the state arrays carry the scratch for that).
 * perm: [n_jobs][epochs][max_rows] int32 row indices relative to the job (shuffle == 2), else NULL.
 * out_loss / out_acc: [n_jobs][epochs] per-epoch sample-weighted mean loss / categorical accuracy
 * (keras History.history["loss"], ["accuracy"], models.py:339-357). */
int gb_ffae_fit(const gb_ffnet* net, float* params, float* adam_m, float* adam_v, const gb_job* jobs,
                int32_t n_jobs, int32_t max_rows, const float* x, const float* y, const int32_t* perm,
                const gb_fit_hparams* hp, float* out_loss, float* out_acc, void* stream);

/* gb_ffae_fit with Keras' validation_split and a row map (a detector that shuffles its rows before the fit).  A job's rows are
 * *positions*: the job trains on positions [0, n_rows) exactly as gb_ffae_fit trains on its rows (sequential order, keyed
 * permutation or `perm` permute positions), and position p reads row x_row + row_map[map_ofs + p] of x and y
 * (x_row + p when map_ofs is -1 or row_map is NULL).  After the last optimizer step of every epoch the job runs the network
 * forward over the held-out positions [n_rows, n_rows + n_val), in order, in batches of val_batch rows, and writes their
 * loss and accuracy, accumulated as the training ones are, to out_val_loss / out_val_acc [n_jobs][epochs]; weights and
 * Adam state are not touched by that pass.  Rows of jobs with n_val 0 are left as they are.  split: [n_jobs] device array,
 * or NULL (no job has held-out positions or a map); several jobs may share one map.  Without a map and held-out
 * positions, the results are those of gb_ffae_fit; with a map, those of gb_ffae_fit on the gathered copy x[map], y[map]. */
typedef struct gb_fit_split {
  int32_t n_val;     /* held-out positions after the job's n_rows training positions */
  int32_t reserved;
  int64_t map_ofs;   /* position p of the job reads row x_row + row_map[map_ofs + p]; -1 = row x_row + p */
} gb_fit_split;

int gb_ffae_fit_split(const gb_ffnet* net, float* params, float* adam_m, float* adam_v, const gb_job* jobs,
                      const gb_fit_split* split, int32_t n_jobs, int32_t max_rows, const float* x, const float* y,
                      const int32_t* row_map, const int32_t* perm, const gb_fit_hparams* hp, int32_t val_batch,
                      float* out_loss, float* out_acc, float* out_val_loss, float* out_val_acc, void* stream);

/* gb_ffae_fit_split with Keras' EarlyStopping callback (keras 3 EarlyStopping.on_epoch_end; models.py EarlyStopping.update), applied
 * by every job at the end of each of its epochs, inside the launch.  The monitored value is the float32 history entry the epoch
 * wrote, widened to double; "better" is v + min_delta < best (mode +1) or v - min_delta > best (mode -1), in double, so a NaN never
 * improves.  Epochs below start_from_epoch are skipped.  With restore_best, the first epoch that is not skipped takes a snapshot,
 * and so does every improvement; `wait` counts the epochs since the last improvement that also beat the baseline; the job stops
 * after the epoch at which wait >= patience and epoch > 0.  At the end, with restore_best and a snapshot, params get the snapshot,
 * whether or not the job stopped early; the Adam state is that of the last epoch run.  A val_* monitor on a job with n_val 0 (or
 * a NULL history array for the monitor) is unavailable: the job never stops and takes no snapshot.
 * stop: [n_jobs] device array, or NULL (then this is gb_ffae_fit_split).  best_params: [n_slots][param_stride], 16-byte aligned,
 * the snapshot area (overwritten where snapshots are taken).  out_epochs: [n_jobs] epochs each job ran; history entries past it
 * are left as they are.  out_best_epoch: [n_jobs] the epoch of the best monitored value (with restore_best: the snapshot's),
 * -1 when no epoch improved and no snapshot was taken.  NULL best_params, out_epochs or out_best_epoch with a stop array, or a
 * misaligned best_params, is GB_E_ARG. */
typedef struct gb_fit_stop {
  int32_t monitor;          /* 0 loss, 1 accuracy, 2 val_loss, 3 val_accuracy */
  int32_t mode;             /* +1 lower is better ("min"), -1 higher is better ("max"); "auto" is resolved by the caller */
  int32_t patience, start_from_epoch;
  int32_t restore_best;     /* the job's final params are those of its best epoch */
  int32_t has_baseline;
  double min_delta;         /* >= 0 */
  double baseline;
} gb_fit_stop;

int gb_ffae_fit_stop(const gb_ffnet* net, float* params, float* adam_m, float* adam_v, const gb_job* jobs,
                     const gb_fit_split* split, int32_t n_jobs, int32_t max_rows, const float* x, const float* y,
                     const int32_t* row_map, const int32_t* perm, const gb_fit_hparams* hp, int32_t val_batch,
                     float* out_loss, float* out_acc, float* out_val_loss, float* out_val_acc, const gb_fit_stop* stop,
                     float* best_params, int32_t* out_epochs, int32_t* out_best_epoch, void* stream);

/* gb_ffae_fit_stop with the optimizer `opt` in place of Adam from hp->lr / beta1 / beta2 / eps.  opt NULL: Adam from hp, bit-identical
 * to gb_ffae_fit_stop; a NULL stop gives gb_ffae_fit_split and a NULL stop and split gb_ffae_fit (out_val_loss, out_val_acc,
 * best_params, out_epochs and out_best_epoch may then be NULL).  hp->lr / beta1 / beta2 / eps are not read when opt is given. */
int gb_ffae_fit_opt(const gb_ffnet* net, float* params, float* adam_m, float* adam_v, const gb_job* jobs,
                    const gb_fit_split* split, int32_t n_jobs, int32_t max_rows, const float* x, const float* y,
                    const int32_t* row_map, const int32_t* perm, const gb_fit_hparams* hp, int32_t val_batch,
                    float* out_loss, float* out_acc, float* out_val_loss, float* out_val_acc, const gb_fit_stop* stop,
                    float* best_params, int32_t* out_epochs, int32_t* out_best_epoch, const gb_optimizer* opt, void* stream);

/* Keras kernel_regularizer / bias_regularizer of Dense layer l (keras 3.3.3 regularizers.L1 / L2 / L1L2 [3P], restated, not verified
 * against TF).  The fit minimises loss + R, R = sum_l kernel_l1[l] sum|W_l| + kernel_l2[l] sum W_l^2 + bias_l1[l] sum|b_l| + bias_l2[l] sum b_l^2,
 * with R evaluated on the weights the step's forward pass uses.  R is part of every mini-batch's total loss, beside the activity
 * term and weighted as it is in the epoch means, so the history, the held-out statistics (R of the current weights) and the
 * EarlyStopping monitor all carry it.  Its gradient l1 sign(w) + 2 l2 w (sign(0) = 0) is added once per optimizer step to the summed
 * mini-batch gradient, before clipvalue and the optimizer's rule; weight decay stays the optimizer's own term. */
typedef struct gb_dense_reg {
  float kernel_l1[GB_MAX_LAYERS], kernel_l2[GB_MAX_LAYERS];
  float bias_l1[GB_MAX_LAYERS], bias_l2[GB_MAX_LAYERS];
} gb_dense_reg;

/* gb_ffae_fit_opt with the weight regularizers `reg`.  reg NULL, or every coefficient 0: exactly gb_ffae_fit_opt (same kernel,
 * bit-identical results).  A negative or non-finite coefficient of a layer of the net is GB_E_ARG, nothing enqueued. */
int gb_ffae_fit_reg(const gb_ffnet* net, float* params, float* adam_m, float* adam_v, const gb_job* jobs,
                    const gb_fit_split* split, int32_t n_jobs, int32_t max_rows, const float* x, const float* y,
                    const int32_t* row_map, const int32_t* perm, const gb_fit_hparams* hp, int32_t val_batch,
                    float* out_loss, float* out_acc, float* out_val_loss, float* out_val_acc, const gb_fit_stop* stop,
                    float* best_params, int32_t* out_epochs, int32_t* out_best_epoch, const gb_optimizer* opt,
                    const gb_dense_reg* reg, void* stream);

/* Keras Dropout(rate) on the input of Dense layer l (keras 3.3.3 layers.Dropout -> tf.nn.dropout [3P], restated, not verified against
 * TF); rate[l] = 0 is the identity, so rate[0] is input dropout and rate[l], l >= 1, drops the activation of layer l-1.  In a training
 * mini-batch, element k of row i of that input becomes keep ? v * s : 0 with s = (float)(1.0 / (1.0 - (double)rate[l])).  The next
 * layer's forward pass, its weight gradient and the reported training loss (and so an EarlyStopping monitor on "loss") read the
 * dropped values; the gradient that flows back through the layer is g * keep * s.  Held-out mini-batches (validation_split) run
 * without dropout, as Keras' evaluation does.  A fresh mask is drawn for every optimizer step.
 * The mask is a stateless counter-based hash, in uint32 arithmetic that wraps, with
 *   mix32(h): h ^= h >> 16; h *= 0x7feb352d; h ^= h >> 15; h *= 0x846ca68b; h ^= h >> 16
 *   key = mix32(lo ^ mix32(hi + 0x632be5ab * (slot + 1)))   lo / hi: low / high 32 bits of hp->seed; slot: the job's gb_job.slot
 *                                                           (the key of the shuffle == 1 permutation)
 *   kd  = mix32(key ^ 0x2545f491)                           the job's dropout key
 *   ks  = mix32(kd + t * 0x9e3779b9)                        t: the absolute 1-based optimizer step of the mini-batch
 *                                                           (hp->step0 + 1 for the first mini-batch of the launch)
 *   kr  = mix32(ks + (p * GB_MAX_LAYERS + l) * 0x85ebca6b)  p: the row's position in its mini-batch, 32 c + r for row r of chunk c
 *   u   = mix32(kr + k * 0x27d4eb2f)                        k: the unit of the input of layer l
 * and the element is kept iff u >= floor(rate[l] * 2^32), computed in double.  Because t counts hp->step0, E one-epoch launches
 * with step0 carried from one to the next draw the masks of one E-epoch launch.  The masks are not Keras' (nor are its initial
 * weights): a Dropout's own seed does not select them. */
typedef struct gb_dense_dropout {
  float rate[GB_MAX_LAYERS];  /* rate on the input of Dense layer l; 0 = none */
} gb_dense_dropout;

/* gb_ffae_fit_reg with dropout `drop`.  drop NULL, or every rate 0: exactly gb_ffae_fit_reg (same kernel, bit-identical results).
 * Invalid (GB_E_ARG, nothing enqueued; the message names the layer): a rate that is negative, >= 1 or not finite; a non-zero rate
 * at l >= net->n_layers; a non-zero rate[l] on the output of a layer with an activity L1 (net->l1[l-1] != 0), whose gradient would
 * need the undropped activation.  The memory plan (gb_ffae_fit_plan) is the same with or without dropout. */
int gb_ffae_fit_drop(const gb_ffnet* net, float* params, float* adam_m, float* adam_v, const gb_job* jobs,
                     const gb_fit_split* split, int32_t n_jobs, int32_t max_rows, const float* x, const float* y,
                     const int32_t* row_map, const int32_t* perm, const gb_fit_hparams* hp, int32_t val_batch,
                     float* out_loss, float* out_acc, float* out_val_loss, float* out_val_acc, const gb_fit_stop* stop,
                     float* best_params, int32_t* out_epochs, int32_t* out_best_epoch, const gb_optimizer* opt,
                     const gb_dense_reg* reg, const gb_dense_dropout* drop, void* stream);

/* The memory plan gb_ffae_fit uses for this architecture (host only, no device needed).  The first of five that fits in
 * 227 KB of shared memory less 2 KB for the fit kernels' static arrays: everything in shared memory; the weight image in the slot's L2-resident state area
 * (*weights_in_l2 = 1); then one, two or three of the three dz buffers there as well (*dz_in_l2).  GB_E_SMEM if none fits
 * (gb_ffae_fit refuses the architecture with the same status); either output may be NULL. */
int gb_ffae_fit_plan(const gb_ffnet* net, int32_t* weights_in_l2, int32_t* dz_in_l2);

/* One architecture of a grouped Dense fit (gb_ffae_fit_group): its net, the state of its slots and its rows.  params, adam_m, adam_v:
 * [this group's slots][param / state stride of net], 16-byte aligned; best_params likewise, needed (and read) only with a stop array.
 * x, y: [rows][net.dims[0]], [rows][net.dims[L]], 16-byte aligned. */
typedef struct gb_fit_group {
  gb_ffnet net;
  float *params, *adam_m, *adam_v, *best_params;
  const float *x, *y;
} gb_fit_group;

/* gb_ffae_fit_drop over jobs of several architectures in one launch.  Job j belongs to group job_group[j] (a HOST array [n_jobs],
 * copied to the device with the group records), and its gb_job.slot, x_row and row ranges are that group's.  Every other argument
 * is gb_ffae_fit_drop's and applies to every job: the jobs, split and stop records, the perm and history rows and out_epochs /
 * out_best_epoch are indexed by the launch's job index, row_map is shared through map_ofs, and hp, opt, reg and drop are every
 * group's.  Each job's results are bit-identical to those of gb_ffae_fit_drop with groups[g].net and its group's pointers over
 * that group's jobs alone: the shuffle permutation and the dropout masks are keyed by (hp->seed, slot), the group-local slot.
 * Refused before any launch (GB_E_ARG unless noted; the message names the group): n_groups < 1; a NULL groups or job_group; a
 * job_group entry outside [0, n_groups); any argument gb_ffae_fit_drop refuses for one group's net and pointers (reg and drop are
 * checked against each group's net); groups whose memory plans (gb_ffae_fit_plan) differ, or whose nets take another kernel
 * family from reg or drop (all-zero coefficients or rates on one net's layers but not another's); a group gb_ffae_fit_drop would
 * refuse (GB_E_SMEM, GB_E_SHAPE, GB_E_ALIGN); a NULL or misaligned workspace.  The dynamic shared memory is the largest of the
 * groups'.  workspace: gb_ffae_fit_group_workspace_bytes(n_groups, n_jobs) bytes of device memory, 16-byte aligned, that the call
 * fills with the group records and job_group (a copy enqueued on `stream`) and the launch reads: it must stay allocated until the
 * launch has run, as any device array of the call. */
size_t gb_ffae_fit_group_workspace_bytes(int32_t n_groups, int32_t n_jobs);
int gb_ffae_fit_group(const gb_fit_group* groups, int32_t n_groups, const int32_t* job_group, const gb_job* jobs,
                      const gb_fit_split* split, int32_t n_jobs, int32_t max_rows, const int32_t* row_map, const int32_t* perm,
                      const gb_fit_hparams* hp, int32_t val_batch, float* out_loss, float* out_acc, float* out_val_loss,
                      float* out_val_acc, const gb_fit_stop* stop, int32_t* out_epochs, int32_t* out_best_epoch,
                      const gb_optimizer* opt, const gb_dense_reg* reg, const gb_dense_dropout* drop, void* workspace,
                      void* stream);

/* ---- K3: LSTM autoencoder predict --------------------------------------------------------
 * lstm_model / lstm_symmetric / lstm_hourglass (factories/lstm_autoencoder.py:72-103):
 * LSTM layers (gate order i,f,c,o; sigmoid recurrent activation; zero initial state per
 * window) then Dense.  Replaces KerasLSTMBaseEstimator.predict (models.py:618-660) without
 * materialising windows (create_keras_timeseriesgenerator, models.py:713-793): output row j
 * of a job is the network applied to x rows [x_row + j, x_row + j + lookback). */
typedef struct gb_lstmnet {
  int32_t n_layers;                 /* LSTM layers */
  int32_t n_features, n_features_out;
  int32_t units[GB_MAX_LAYERS];
  int32_t act[GB_MAX_LAYERS];       /* cell/output activation of each LSTM layer (tanh default) */
  int32_t out_act;                  /* Dense activation */
  int32_t lookback;
} gb_lstmnet;

/* per-slot parameter vector: for each layer: kernel [in][4u], recurrent_kernel [u][4u], bias [4u];
 * then Dense kernel [u_last][n_out], bias [n_out]. */
size_t gb_lstm_param_count(const gb_lstmnet* net);
size_t gb_lstm_param_stride(const gb_lstmnet* net);
/* jobs: n_rows = number of *windows* (output rows); x rows read = n_rows + lookback - 1.
 * workspace: gb_lstm_workspace_bytes() bytes of device scratch. */
size_t gb_lstm_workspace_bytes(const gb_lstmnet* net, int32_t n_jobs, int32_t max_rows);
int gb_lstm_infer(const gb_lstmnet* net, const float* params, const gb_job* jobs, int32_t n_jobs,
                  int32_t max_rows, const float* x, float* out_model, void* workspace, void* stream);

/* ---- K3 on the tensor cores, wgmma (layer widths 1..512, padded to multiples of 64 internally; tanh and sigmoid cells
 * only, since h is carried as an FP16 pair and a relu or linear cell's h is unbounded).  One launch per
 * (layer, timestep) advances every window of every job: [h_below,t | h_own,t-1] . [K; U]^T on the tensor cores
 * (FP16-pair split operands, fp32 accumulation), LSTM cell in the epilogue, recurrent state in `workspace`
 * (gb_lstm_tc_workspace_bytes; x_rows = rows of the x array, n_slots = rows of params). */
int gb_lstm_tc_supported(const gb_lstmnet* net);
size_t gb_lstm_tc_workspace_bytes(const gb_lstmnet* net, int32_t n_slots, int32_t n_jobs, int32_t max_windows, int64_t x_rows);
int gb_lstm_infer_tc(const gb_lstmnet* net, const float* params, int32_t n_slots, const gb_job* jobs, int32_t n_jobs,
                     int32_t max_windows, const float* x, int64_t x_rows, float* out_model, void* workspace, void* stream);
/* The same kernels over a ragged tile layout, for jobs of very different lengths (a request coalescer's batch): job j's windows
 * occupy the flat 128-window tiles [tile_base[j], tile_base[j + 1]), so the recurrent state, the input projection and the work
 * grow with the jobs' own windows, not with n_jobs x the longest job.  tile_base: DEVICE array of n_jobs + 1 int32, the prefix sums
 * of ceil(n_rows_j / 128) (tile_base[0] = 0, tile_base[n_jobs] = n_tiles); max_windows >= every job's n_rows, and n_tiles <=
 * n_jobs * ceil(max_windows / 128).  Each window's arithmetic is that of gb_lstm_infer_tc, so its output is the same bits in
 * either entry and any batch.  workspace: gb_lstm_tc_ragged_workspace_bytes() bytes (0 for arguments it refuses). */
size_t gb_lstm_tc_ragged_workspace_bytes(const gb_lstmnet* net, int32_t n_slots, int32_t n_jobs, int32_t n_tiles, int32_t max_windows);
int gb_lstm_infer_tc_ragged(const gb_lstmnet* net, const float* params, int32_t n_slots, const gb_job* jobs, int32_t n_jobs,
                            const int32_t* tile_base, int32_t n_tiles, int32_t max_windows, const float* x, int64_t x_rows,
                            float* out_model, void* workspace, void* stream);

/* ---- K3-fit: LSTM training (back-propagation through time) ---------------------------------
 * Replaces KerasLSTMBaseEstimator.fit (models.py:557-616): if `primer`, one Adam step on the single
 * window 0 (the reference's `super().fit` on a batch of one, :585-597); then `epochs` passes over the
 * windows in order (shuffle=False, :612-615) in batches of `batch_size` (last partial batch kept),
 * loss = mean((net(window) - target)^2), Adam as in gb_ffae_fit.  Window j of a job = x rows
 * [x_row + j, x_row + j + lookback), target = y row x_row + j + lookback - 1 + lookahead; jobs[].n_rows
 * counts windows.  params / adam_m / adam_v: [n_slots][gb_lstm_param_stride], updated in place;
 * adam_t: [n_slots] optimizer step counters (in/out).  out_loss / out_acc: [n_jobs][epochs].
 * workspace: gb_lstm_fit_workspace_bytes(net, n_jobs) bytes of device scratch (saved gates/states of
 * one batch per job).  One optimizer step is a sequence of launches over (tile, job) grids. */
typedef struct gb_lstm_fit_hparams {
  int32_t epochs, batch_size;   /* batch_size <= 32 (gb_lstm_fit_tc: <= 256) */
  int32_t lookahead;            /* 0 = KerasLSTMAutoEncoder, 1 = KerasLSTMForecast */
  int32_t primer;               /* 1 = run the reference's primer step first */
  float lr, beta1, beta2, eps;
} gb_lstm_fit_hparams;
size_t gb_lstm_fit_workspace_bytes(const gb_lstmnet* net, int32_t n_jobs);
int gb_lstm_fit(const gb_lstmnet* net, float* params, float* adam_m, float* adam_v, int32_t* adam_t,
                const gb_job* jobs, int32_t n_jobs, int32_t max_windows, const float* x, const float* y,
                const gb_lstm_fit_hparams* hp, void* workspace, float* out_loss, float* out_acc, void* stream);
/* gb_lstm_fit on the gb_loss `loss` (primer step and history included): loss = mean(f(net(window), target)).
 * gb_lstm_fit is this with GB_LOSS_MSE.  Outside 0..5: GB_E_ARG, nothing enqueued. */
int gb_lstm_fit_loss(const gb_lstmnet* net, float* params, float* adam_m, float* adam_v, int32_t* adam_t,
                     const gb_job* jobs, int32_t n_jobs, int32_t max_windows, const float* x, const float* y,
                     const gb_lstm_fit_hparams* hp, void* workspace, float* out_loss, float* out_acc, int32_t loss,
                     void* stream);
/* gb_lstm_fit_loss for batches of 1..256 windows, on the tensor cores: the same steps, order, losses, history and Adam state,
 * with the GEMMs of a step (forward gates, backward input, weight gradients) on wgmma in split TF32 (hi*hi + hi*lo + lo*hi,
 * fp32 accumulation) over 64-window batch tiles.  workspace: gb_lstm_fit_tc_workspace_bytes(net, n_jobs, batch_size) bytes
 * (grows with the batch rounded up to 64, x lookback x the units; 0 for an invalid net or batch_size outside 1..256).
 * batch_size > 256: GB_E_SHAPE, nothing enqueued. */
size_t gb_lstm_fit_tc_workspace_bytes(const gb_lstmnet* net, int32_t n_jobs, int32_t batch_size);
int gb_lstm_fit_tc(const gb_lstmnet* net, float* params, float* adam_m, float* adam_v, int32_t* adam_t,
                   const gb_job* jobs, int32_t n_jobs, int32_t max_windows, const float* x, const float* y,
                   const gb_lstm_fit_hparams* hp, void* workspace, float* out_loss, float* out_acc, int32_t loss,
                   void* stream);
/* gb_lstm_fit_loss / gb_lstm_fit_tc with the gb_optimizer `opt` in place of Adam from hp->lr / beta1 / beta2 / eps (adam_m / adam_v
 * are its state slots 0 / 1, adam_t its step counts).  opt NULL: Adam from hp, bit-identical to the entry point without _opt. */
int gb_lstm_fit_opt(const gb_lstmnet* net, float* params, float* adam_m, float* adam_v, int32_t* adam_t,
                    const gb_job* jobs, int32_t n_jobs, int32_t max_windows, const float* x, const float* y,
                    const gb_lstm_fit_hparams* hp, void* workspace, float* out_loss, float* out_acc, int32_t loss,
                    const gb_optimizer* opt, void* stream);
int gb_lstm_fit_tc_opt(const gb_lstmnet* net, float* params, float* adam_m, float* adam_v, int32_t* adam_t,
                       const gb_job* jobs, int32_t n_jobs, int32_t max_windows, const float* x, const float* y,
                       const gb_lstm_fit_hparams* hp, void* workspace, float* out_loss, float* out_acc, int32_t loss,
                       const gb_optimizer* opt, void* stream);
/* gb_lstm_fit_opt / gb_lstm_fit_tc_opt with Keras' EarlyStopping callback (keras 3 EarlyStopping.on_epoch_end; models.py
 * EarlyStopping.update), applied by every job at the end of each of its epochs, inside the call, as the per-machine fit loop applies
 * it after each one-epoch launch (the primer step is not an epoch; epochs count from 0).  The monitored value is the float32
 * history entry the epoch wrote, widened to double; "better" is v + min_delta < best (mode +1) or v - min_delta > best (mode -1),
 * in double, so a NaN never improves.  Epochs below start_from_epoch are skipped.  With restore_best, the first epoch that is not
 * skipped takes a snapshot, and so does every improvement; `wait` counts the epochs since the last improvement that also beat the
 * baseline; the job stops after the epoch at which wait >= patience and epoch > 0.  From then on it does no work: its params,
 * optimizer state and step count stay as the last epoch it ran left them, and once every job has stopped the remaining steps
 * skip their kernels.  At the end, with restore_best and a snapshot, params get the snapshot, whether or not the job stopped
 * early; the optimizer state is that of the last epoch run.  The LSTM fit reports loss and accuracy only, so a val_* monitor
 * (2, 3) is unavailable: the job never stops and takes no snapshot.
 * stop: [n_jobs] *host* array of gb_fit_stop, read before the call returns, or NULL (then this is the _opt entry point, bit for
 * bit).  With a stop array the workspace is gb_lstm_fit_workspace_bytes(net, n_jobs) (gb_lstm_fit_tc_stop:
 * gb_lstm_fit_tc_workspace_bytes(net, n_jobs, batch_size)) + gb_lstm_fit_stop_state_bytes(n_jobs) bytes: the rule's per-job
 * state lives at its end.  best_params: [n_slots][param_stride] device, 16-byte aligned, the snapshot area (overwritten where
 * snapshots are taken).  out_epochs: [n_jobs] device, epochs each job ran; history entries past it are left as they are.
 * out_best_epoch: [n_jobs] device, the epoch of the best monitored value (with restore_best: the snapshot's), -1 when no epoch
 * improved and no snapshot was taken.  GB_E_ARG, nothing enqueued and no device needed: NULL best_params, out_epochs or
 * out_best_epoch with a stop array, a misaligned best_params, a monitor outside 0..3, a mode other than +1 / -1, a negative
 * patience or a negative min_delta. */
size_t gb_lstm_fit_stop_state_bytes(int32_t n_jobs);
int gb_lstm_fit_stop(const gb_lstmnet* net, float* params, float* adam_m, float* adam_v, int32_t* adam_t,
                     const gb_job* jobs, int32_t n_jobs, int32_t max_windows, const float* x, const float* y,
                     const gb_lstm_fit_hparams* hp, void* workspace, float* out_loss, float* out_acc, int32_t loss,
                     const gb_optimizer* opt, const gb_fit_stop* stop, float* best_params, int32_t* out_epochs,
                     int32_t* out_best_epoch, void* stream);
int gb_lstm_fit_tc_stop(const gb_lstmnet* net, float* params, float* adam_m, float* adam_v, int32_t* adam_t,
                        const gb_job* jobs, int32_t n_jobs, int32_t max_windows, const float* x, const float* y,
                        const gb_lstm_fit_hparams* hp, void* workspace, float* out_loss, float* out_acc, int32_t loss,
                        const gb_optimizer* opt, const gb_fit_stop* stop, float* best_params, int32_t* out_epochs,
                        int32_t* out_best_epoch, void* stream);

/* Keras' Orthogonal initialiser for recurrent kernels: g holds n_mats standard-normal [rows][cols] draws (float64, rows <= cols,
 * overwritten); matrix i's rows are orthonormalised (Gram-Schmidt, the sign convention of Keras' QR) and written as float32 to
 * out + out_offset + i * out_stride, row-major. */
int gb_orthonormal_rows(double* g, int32_t n_mats, int32_t rows, int32_t cols, float* out, int64_t out_offset, int64_t out_stride,
                        void* stream);

#ifdef __cplusplus
}
#endif
#endif /* GORDO_B200_H */
