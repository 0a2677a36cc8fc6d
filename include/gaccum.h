/* gaccum.h -- C ABI of libgaccum.so: the H100 (sm_90a) gradient-accumulation train_op.
 *
 * This is the drop-in boundary for ONE path of hpandana/gradient-accumulation-tf-estimator:
 * the accumulate-then-apply train_op that `create_optimizer` builds
 * (reference optimization.py:25-104) together with `AdamWeightDecayOptimizer.apply_gradients`
 * (optimization.py:128-177) and the plain-Adam variant the distributedExample scripts inline
 * (02_single_worker_with_estimator_gaccum.py:47-73, 04_multi_worker_with_estimator_gaccum.py:48-74,
 * another-example.py:126-155).  Each entry point cites the reference lines it replaces.
 *
 * Conventions
 *   - plain C types only; every function returns 0 on success or a negative GACCUM_E* code
 *     (helpers that return a value say so); `gaccum_last_error()` gives a thread-local message.
 *   - the caller owns every device buffer (params, grads, accum, m, v); the library owns only
 *     the opaque plan (static tile table, decay mask, per-CTA partial buffer, stats block).
 *   - all hot calls are asynchronous on the caller's CUDA stream, never synchronise the host,
 *     and launch exactly one kernel (the data-parallel apply step included).  A plan may be used
 *     on one stream at a time.
 *   - there is NO CPU fallback: without a CUDA device every compute call fails with
 *     GACCUM_ENODEVICE.  A plan created with device = -1 is layout-only (offset queries).
 *   - all state is IEEE fp32; arithmetic follows the reference's un-fused op order with
 *     round-to-nearest on every op (no FMA contraction), so results are bit-identical to the
 *     oracle whenever the clip scale is exactly 1 (see DESIGN.md "Numerics").
 */
#ifndef GACCUM_H_
#define GACCUM_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define GACCUM_API __attribute__((visibility("default")))
#else
#define GACCUM_API
#endif

#define GACCUM_VERSION 200 /* 0.2.0: TMA-fed clip-apply, push-based data-parallel apply (gaccum_dp_comm changed) */

/* error codes */
#define GACCUM_OK 0
#define GACCUM_EINVAL (-1)    /* bad argument (message says which) */
#define GACCUM_ENODEVICE (-2) /* no CUDA device / layout-only plan used for compute */
#define GACCUM_ECUDA (-3)     /* a CUDA runtime call failed */
#define GACCUM_ENCCL (-4)     /* NCCL missing or an NCCL call failed */
#define GACCUM_ENOMEM (-5)

/* optimizer variants */
#define GACCUM_ADAM_WEIGHT_DECAY 0 /* optimization.py:107-194 (BERT path; "variant A") */
#define GACCUM_ADAM 1              /* tf.train.AdamOptimizer, TF1 ApplyAdam (02:41,61; 04:42,62) */

typedef struct gaccum_plan gaccum_plan;
typedef void* gaccum_stream_t; /* a cudaStream_t */

/* Hyper-parameters the reference hard-codes.  Doubles because the reference passes Python
 * floats and converts to fp32 at specific points (e.g. `1.0 - self.beta_1` is evaluated in
 * double first, optimization.py:152). */
typedef struct gaccum_hparams {
  int32_t variant;          /* GACCUM_ADAM_WEIGHT_DECAY | GACCUM_ADAM */
  int32_t reserved;         /* must be 0 */
  double beta1;             /* optimization.py:62  (0.9)  */
  double beta2;             /* optimization.py:63  (0.999) */
  double epsilon;           /* optimization.py:64  (1e-6); tf.train.AdamOptimizer: 1e-8 */
  double weight_decay_rate; /* optimization.py:61  (0.01); ignored by GACCUM_ADAM */
  double clip_norm;         /* optimization.py:84  (1.0); <= 0 disables tf.clip_by_global_norm */
} gaccum_hparams;

/* Per-micro-step scalars (the values the TF graph would feed the op as host tensors). */
typedef struct gaccum_step_args {
  int64_t global_step; /* PRE-increment tf.train.get_global_step() value, optimization.py:27,77 */
  int32_t accum_n;     /* gradient_accumulation_multiplier, optimization.py:76 */
  int32_t reserved;    /* must be 0 */
  float lr;            /* learning rate of this micro-step (gaccum_learning_rate) */
  float beta1_power;   /* GACCUM_ADAM only: TF1 Adam non-slot variable, beta1^t, t = #applies+1 */
  float beta2_power;   /* GACCUM_ADAM only */
  float reserved2;     /* must be 0 */
} gaccum_step_args;

/* What the last step on this plan computed (device-written, read back with gaccum_read_stats). */
typedef struct gaccum_stats {
  float applied;     /* 1 if the step took the apply branch of the tf.cond (optimization.py:91) */
  float lr;          /* lr used */
  float global_norm; /* tf.linalg.global_norm of the normalised accumulators (0 when not clipping) */
  float clip_scale;  /* the scalar tf.clip_by_global_norm multiplies by (1 when not clipping) */
} gaccum_stats;

/* ---- library -------------------------------------------------------------------------- */
GACCUM_API int gaccum_version(void);
GACCUM_API const char* gaccum_last_error(void);
/* number of visible CUDA devices (0 when there is no driver/GPU); never fails */
GACCUM_API int gaccum_device_count(void);

/* ---- host-side scalar logic of the reference graph ------------------------------------ */
/* optimization.py:29-54: polynomial decay (power 1, end 0) + linear warm-up, fp32 op order.
 * num_warmup_steps == 0 means "no warm-up" (the reference's `if num_warmup_steps:`). */
GACCUM_API float gaccum_learning_rate(double init_lr, int64_t num_train_steps,
                                      int64_t num_warmup_steps, int64_t global_step);
/* optimization.py:77,91: the tf.cond predicate, int32(global_step) % N == 0 (pre-increment). */
GACCUM_API int gaccum_is_apply_step(int64_t global_step, int32_t accum_n);
/* optimization.py:179-194: decay mask from variable names.  `exclude` are regular expressions
 * searched in the name; a trailing ":<digits>" is stripped from each name first.
 * out[i] = 1 iff tensor i gets weight decay.
 * DIALECT: POSIX extended (regcomp REG_EXTENDED), the reference uses Python `re.search`
 * (optimization.py:185).  The two agree on the reference's own patterns ("LayerNorm",
 * "layer_norm", "bias" -- plain substrings) and on the common subset; Python-only syntax
 * (\d, \w, look-arounds, non-greedy) is rejected with GACCUM_EINVAL or matches differently.
 * Callers that accept user patterns should evaluate them with the reference's engine and pass
 * the resulting mask to gaccum_plan_create -- both Python bindings in this repository do. */
GACCUM_API int gaccum_decay_mask(int32_t num_tensors, const char* const* names,
                                 double weight_decay_rate, const char* const* exclude,
                                 int32_t num_exclude, uint8_t* out);

/* ---- plan ----------------------------------------------------------------------------- */
/* Describes the T trainable tensors (tf.trainable_variables() order, optimization.py:70) and
 * lays out the packed fp32 slabs that replace the per-variable `accum_grads` (optimization.py:78)
 * and `adam_m` / `adam_v` (optimization.py:137-148).  device = -1: layout-only plan. */
GACCUM_API int gaccum_plan_create(gaccum_plan** out, int32_t num_tensors, const int64_t* numels,
                                  const uint8_t* decay, const gaccum_hparams* hp, int32_t device);
GACCUM_API int gaccum_plan_destroy(gaccum_plan* plan);
/* elements (not bytes) each of the accum / m / v slabs must hold */
GACCUM_API int64_t gaccum_padded_size(const gaccum_plan* plan);
/* out[i] = element offset of tensor i inside a slab (multiples of 32 elements = 128 B) */
GACCUM_API int gaccum_offsets(const gaccum_plan* plan, int64_t* out);
GACCUM_API int32_t gaccum_num_tensors(const gaccum_plan* plan);
GACCUM_API int64_t gaccum_num_elements(const gaccum_plan* plan); /* P, real elements */
GACCUM_API int32_t gaccum_num_tiles(const gaccum_plan* plan);
/* Algorithmic bytes of one launch: accumulate = 12 B x P; apply = 36 B x P (SURVEY.md 8(d)). */
GACCUM_API int64_t gaccum_algorithmic_bytes(const gaccum_plan* plan, int32_t is_apply);

/* ---- the hot path --------------------------------------------------------------------- */
/* One micro-step of the train_op (optimization.py:91-94): if gaccum_is_apply_step() the apply
 * branch (assign_add -> /N -> clip_by_global_norm -> apply_gradients -> zero; :80-88), else
 * the accumulate branch (:93).  grads[i] / params[i]: device pointers to tensor i (scattered,
 * any 4-byte alignment; 16-byte alignment takes the vector path).  grads[i] == NULL means
 * "no gradient for this tensor" (optimization.py:132 skips such pairs).
 * accum / m / v: device slabs of gaccum_padded_size() floats, 16-byte aligned.
 * The caller increments global_step afterwards (optimization.py:102-103). */
GACCUM_API int gaccum_step(gaccum_plan* plan, const float* const* grads, float* const* params,
                           float* accum, float* m, float* v, const gaccum_step_args* args,
                           gaccum_stream_t stream);
/* The two branches on their own (the data-parallel driver accumulates locally, all-reduces the
 * slab, then applies with grads == NULL).  gaccum_apply ignores args->global_step. */
GACCUM_API int gaccum_accumulate(gaccum_plan* plan, const float* const* grads, float* accum,
                                 gaccum_stream_t stream);
GACCUM_API int gaccum_apply(gaccum_plan* plan, const float* const* grads, float* const* params,
                            float* accum, float* m, float* v, const gaccum_step_args* args,
                            gaccum_stream_t stream);
/* Same step when gradients and parameters are themselves packed in slab layout (params as
 * views of one flat buffer): no pointer table.  grad_slab may be NULL on an apply step. */
GACCUM_API int gaccum_step_packed(gaccum_plan* plan, const float* grad_slab, float* param_slab,
                                  float* accum, float* m, float* v, const gaccum_step_args* args,
                                  int32_t force_branch /* -1 = from global_step, 0 = accumulate, 1 = apply */,
                                  gaccum_stream_t stream);
/* ---- data parallel: the apply step fused with its exchange over NVLink peer memory ------- */
/* Replaces reference distributedExample/04's MultiWorkerMirroredStrategy wiring: accumulators
 * with aggregation=SUM (04:55) all-reduced per variable on every micro-step (04:58,70) and a
 * replicated apply (04:59-66).  Each rank calls gaccum_step_dp once per micro-step: accumulate
 * steps are the rank-local accumulate kernel (no bytes cross NVLink); the apply step is ONE kernel
 * (csrc/gaccum_dp.cuh) that adds the last gradient, pushes every foreign tile of a + G into its
 * owner's staging area (reduce-scatter by peer stores), reduces its own shard in fixed rank order,
 * exchanges the partial global norms, updates the tiles the rank owns and pushes the new parameters
 * into every rank's parameter slab (all-gather by peer stores).  The loss is expected to be
 * pre-divided by the number of workers, as 04:46 does. */
#define GACCUM_MAX_RANKS 8
#define GACCUM_DP_CTRL_BYTES 256
typedef struct gaccum_dp_comm {
  int32_t rank;
  int32_t world; /* 2..GACCUM_MAX_RANKS */
  /* this rank's packed fp32 accumulator slab (gaccum_padded_size floats); private, never peer-accessed */
  float* accum;
  /* Base device pointers of every rank's buffers, all mapped into this process (symmetric
   * memory / CUDA IPC / cuMem fabric handles); entry [rank] is the local buffer.
   *   param_peers: packed fp32 parameter slabs, slab layout (gaccum_offsets)
   *   stage_peers: staging areas of gaccum_dp_stage_elements() floats (contents are scratch)
   *   ctrl_peers : GACCUM_DP_CTRL_BYTES control blocks, zero-initialised once */
  float* param_peers[GACCUM_MAX_RANKS];
  float* stage_peers[GACCUM_MAX_RANKS];
  uint32_t* ctrl_peers[GACCUM_MAX_RANKS];
  int64_t stage_elements; /* floats each staging area holds */
} gaccum_dp_comm;
/* tiles [*tile_lo, *tile_hi) and the element count rank `rank` of `world` owns */
GACCUM_API int gaccum_dp_shard_range(const gaccum_plan* plan, int32_t world, int32_t rank,
                                     int32_t* tile_lo, int32_t* tile_hi, int64_t* num_elements);
/* floats every rank's staging area must hold for `world` ranks: (world-1) x the widest shard */
GACCUM_API int64_t gaccum_dp_stage_elements(const gaccum_plan* plan, int32_t world);
/* One micro-step on this rank (04:48-74).  grads[i]: this rank's gradient of tensor i (device, scattered,
 * NULL = none).  `epoch` must be non-zero, different from the previous apply's (e.g. an apply counter)
 * and the same on every rank.  m / v: local slabs; only the owned range is read or written.
 * All `world` ranks must call this for the same step; the call is asynchronous on `stream`.
 * If a peer never reaches the matching apply (crashed rank, mismatched epoch) the kernel traps after
 * 60 s of waiting and the failure surfaces as a CUDA error on the next runtime call. */
GACCUM_API int gaccum_step_dp(gaccum_plan* plan, const gaccum_dp_comm* comm, const float* const* grads,
                              float* m, float* v, const gaccum_step_args* args, uint32_t epoch,
                              gaccum_stream_t stream);
/* the apply branch alone (args->global_step is not consulted) */
GACCUM_API int gaccum_apply_dp(gaccum_plan* plan, const gaccum_dp_comm* comm, const float* const* grads,
                               float* m, float* v, const gaccum_step_args* args, uint32_t epoch,
                               gaccum_stream_t stream);

/* ---- host-buffer session: the same train_op for a caller whose tensors live in HOST memory -- */
/* (e.g. the reference run with CPU placement, distributedExample/02 "1 worker CPU").  The session
 * keeps params / accum / m / v resident in HBM in packed layout; every micro-step copies that
 * step's gradients host->device (double-buffered on a private copy stream so the copy of step k+1
 * overlaps the kernel of step k), launches the one kernel, and on apply steps copies the updated
 * parameters device->host.  Pinned host memory makes the copies truly asynchronous.
 * gaccum_step_host returns after enqueueing; gaccum_host_session_sync waits for completion. */
typedef struct gaccum_host_session gaccum_host_session;
GACCUM_API int gaccum_host_session_create(gaccum_host_session** out, gaccum_plan* plan);
GACCUM_API int gaccum_host_session_destroy(gaccum_host_session* s);
/* initial values of the trainable variables (optimization.py:70) -> HBM; synchronous */
GACCUM_API int gaccum_host_session_set_params(gaccum_host_session* s, const float* const* host_params);
/* host_grads[i] may be NULL (no gradient).  host_params_out (may be NULL) receives the updated
 * parameters on apply steps.  stats_out (may be NULL) receives the stats block every step. */
GACCUM_API int gaccum_step_host(gaccum_host_session* s, const float* const* host_grads,
                                float* const* host_params_out, const gaccum_step_args* args,
                                gaccum_stats* stats_out);
GACCUM_API int gaccum_host_session_sync(gaccum_host_session* s);
/* Copies are coalesced: a run of tensors whose host addresses are spaced like their slab offsets
 * (gaccum_offsets; padding included) moves with ONE cudaMemcpyAsync, so a caller that keeps its
 * gradients / parameters in a pinned arena with the plan's layout pays one copy per direction.
 *
 * Data parallel over host buffers (reference 04 with CPU-resident tensors): every rank creates a
 * session, calls _dp_export, the caller exchanges the records between the ranks with whatever
 * transport it has (MPI, torch.distributed, TF collectives -- they are plain bytes), every rank calls
 * _dp_connect with all of them.  From then on the apply step of gaccum_step_host is the fused
 * exchange + apply kernel of gaccum_apply_dp over CUDA-IPC peer mappings of the other ranks'
 * parameter slabs / staging areas; accumulate steps stay rank-local.  All ranks must step in
 * lock-step (same global_step, same accum_n).  Ranks must be GPUs of one peer-access domain. */
#define GACCUM_IPC_HANDLE_BYTES 64
typedef struct gaccum_dp_ipc {
  unsigned char param[GACCUM_IPC_HANDLE_BYTES]; /* cudaIpcMemHandle_t of the parameter slab */
  unsigned char stage[GACCUM_IPC_HANDLE_BYTES]; /* ... of the reduce-scatter staging area */
  unsigned char ctrl[GACCUM_IPC_HANDLE_BYTES];  /* ... of the control block */
  int64_t stage_elements;
  int64_t padded_size;
} gaccum_dp_ipc;
GACCUM_API int gaccum_host_session_dp_export(gaccum_host_session* s, int32_t world, gaccum_dp_ipc* out);
GACCUM_API int gaccum_host_session_dp_connect(gaccum_host_session* s, int32_t rank, int32_t world,
                                              const gaccum_dp_ipc* all /* world records, rank order */);
/* device pointers of the resident slabs (params, accum, m, v) for inspection: out[4] */
GACCUM_API int gaccum_host_session_slabs(gaccum_host_session* s, float** out);

/* Asynchronously copy the stats block of the last step to host memory (pinned for true async). */
GACCUM_API int gaccum_read_stats(gaccum_plan* plan, gaccum_stats* host_out, gaccum_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* GACCUM_H_ */
