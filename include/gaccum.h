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
#define GACCUM_LAMB 2              /* LAMB (You et al. 2019, "Large Batch Optimization for Deep Learning"), see below */

/* GACCUM_LAMB, in the form of TF-Addons' LAMB with the fp32 op order of GACCUM_ADAM_WEIGHT_DECAY (one correctly rounded
 * op per TF op, no FMA contraction).  It uses the same hyper-parameters as AdamWeightDecay.  The apply step's prelude is
 * unchanged: c = (1.0 * a') / N, times 1/S under loss scaling, times the clip scale.  Then, per tensor:
 *     m  = b1*m + omb1*c            v  = b2*v + omb2*(c*c)      omb = fp32(1.0 - beta) from double, as variant A
 *     mh = m / (1 - beta1_power)    vh = v / (1 - beta2_power)  fp32 ops
 *     u  = mh / (sqrt(vh) + eps)
 *     if decay[i]:  u = u + wd*p
 *     r  = 1
 *     if adapt[i]:  wn = ||p||, un = ||u||   (p before the update; ||x|| = sqrtf(fp32(sum x^2)))
 *                   r  = (wn > 0 && un > 0) ? wn / un : 1
 *     p  = p - (r*lr)*u              the scalar product first, as `ratio * lr * update` evaluates (lr: the tensor's lr_t
 *                                    with gaccum_plan_set_lr_multipliers)
 * The beta powers are TF1 Adam's running fp32 products (beta_power *= beta after every APPLIED window, starting at
 * fp32(beta)), not pow(beta, t): gaccum_step_args.beta{1,2}_power, or under loss scaling the device block's, which the
 * apply advances on windows it does not skip.  decay[] is gaccum_plan_create's mask; adapt[] is set with
 * gaccum_plan_set_layer_adaptation (default: every tensor adapts).  The sums of squares are exact (fixed-point
 * accumulation of fp64 partials, independent of the work split) and rounded to fp32 once, so r is deterministic from run
 * to run; it can differ in the last bit from a plain fp64 sum.  Everything else -- the pre-increment predicate, the
 * first-accumulate precondition, tensors without a gradient, stats, the loss-scaling skip (a = +0 only; p, m, v, the
 * master weights, the model copy and the beta powers unchanged bit for bit) -- is as for AdamWeightDecay.
 * gaccum_step_dp, gaccum_apply_dp, gaccum_host_session_create and gaccum_step_host refuse a LAMB plan with
 * GACCUM_EINVAL. */

/* element types of the model's weights and gradients (gaccum_plan_set_param_dtype) */
#define GACCUM_DTYPE_F32 0  /* the default: no call needed */
#define GACCUM_DTYPE_BF16 1
#define GACCUM_DTYPE_F16 2

typedef struct gaccum_plan gaccum_plan;
typedef void* gaccum_stream_t; /* a cudaStream_t */

/* Hyper-parameters the reference hard-codes.  Doubles because the reference passes Python
 * floats and converts to fp32 at specific points (e.g. `1.0 - self.beta_1` is evaluated in
 * double first, optimization.py:152). */
typedef struct gaccum_hparams {
  int32_t variant;          /* GACCUM_ADAM_WEIGHT_DECAY | GACCUM_ADAM | GACCUM_LAMB */
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
  float beta1_power;   /* GACCUM_ADAM, GACCUM_LAMB: TF1 Adam non-slot variable, beta1^t, t = #applies+1 */
  float beta2_power;   /* GACCUM_ADAM, GACCUM_LAMB */
  float reserved2;     /* must be 0 */
} gaccum_step_args;

/* What the last step on this plan computed (device-written, read back with gaccum_read_stats). */
typedef struct gaccum_stats {
  float applied;     /* 1 if the step took the apply branch of the tf.cond (optimization.py:91) */
  float lr;          /* lr used */
  float global_norm; /* tf.linalg.global_norm of the normalised accumulators (0 when not clipping) */
  float clip_scale;  /* the scalar tf.clip_by_global_norm multiplies by (1 when not clipping) */
} gaccum_stats;

/* Dynamic loss scaling for fp16 mixed precision (TF 2's DynamicLossScale, counted in windows).  The producer computes
 * gradients of loss * S, so the accumulators hold sums of S * g.  The apply step unscales, c = ((1.0 * a') / N) * (1/S),
 * and skips the window -- a = +0.0 everywhere, p, m, v (and GACCUM_ADAM's beta powers) unchanged bit for bit -- when an
 * element of a' is not finite or, with clipping on, the global norm is not.  Then, on a skipped window,
 * S = max(1, S / multiplier) and good_windows = 0; on an applied one, if good_windows + 1 >= growth_interval,
 * S = S * multiplier (only if that is finite) and good_windows = 0, else good_windows += 1.  S is always a power of two,
 * so the unscale is exact and a run whose scaled values stay normal fp32 numbers is bit-identical to the same run
 * without loss scaling fed unscaled gradients.  Accumulate steps are unchanged. */
typedef struct gaccum_loss_scale_config {
  double initial_scale;    /* a power of two in [1, 2^127] */
  double multiplier;       /* a power of two in [2, 2^127] (TF 2: 2) */
  int32_t growth_interval; /* >= 1: applied windows before S grows (TF 2: 2000) */
  int32_t reserved;        /* must be 0 */
} gaccum_loss_scale_config;

/* The loss-scaling state: 32 bytes of caller-owned DEVICE memory (16-byte aligned), written by
 * gaccum_loss_scale_init and afterwards only by the apply launches, so no step needs the host.  A producer may read
 * `scale` on the device (e.g. multiply its loss by it) between steps. */
typedef struct gaccum_loss_scale_state {
  float scale;              /* S */
  int32_t good_windows;     /* applied windows since S last changed */
  uint32_t skipped_windows; /* overflowed windows since gaccum_loss_scale_init */
  int32_t last_skipped;     /* 1 if the last apply step skipped its window, else 0 */
  float beta1_power;        /* GACCUM_ADAM, GACCUM_LAMB: TF1's beta1^t, used instead of gaccum_step_args.beta1_power and */
  float beta2_power;        /*   advanced (one fp32 multiply each) on applied windows only */
  float reserved[2];
} gaccum_loss_scale_state;

/* An exponential moving average of the weights, kept by the apply step (TF1 tf.train.ExponentialMovingAverage with
 * zero_debias=False, applied once per APPLIED window -- `with tf.control_dependencies([train_op]): ema.apply(tvars)`
 * without its pull toward unchanged weights on every micro-step).  Every step is one correctly rounded fp32 op, no FMA:
 *     d = fp32(decay)
 *     num_updates mode:  nf = fp32(n);  d = min(d, (1 + nf) / (10 + nf))      (fp32 add, add, div, min)
 *     c = 1 - d                                                                (fp32 subtract)
 *     e = e - (e - p) * c                                                      (fp32 sub, mul, sub)
 * p is the value the apply just stored: the parameter, or the fp32 master weight of a 16-bit plan.  Every tensor is
 * averaged, tensors without a gradient in the window included; accumulate steps do not touch the average.  n is the
 * number of windows averaged before this one: it lives in the device state and the apply advances it, so a captured
 * graph replayed k times advances it k times.  A window that loss scaling skips leaves the average and the state
 * unchanged bit for bit.  Nothing the training computes (p, m, v, accumulators, stats, trust ratios, the loss-scaling
 * state, the model copy) depends on whether an average is kept.  The caller initialises the average, as TF initialises
 * a shadow variable to its variable's value. */
typedef struct gaccum_ema_config {
  double decay;          /* in [0, 1] (TF: e.g. 0.9999) */
  int32_t num_updates;   /* 0, or 1: TF's num_updates warm-up d = min(decay, (1 + n) / (10 + n)) */
  int32_t reserved;      /* must be 0 */
} gaccum_ema_config;

/* The EMA state: 16 bytes of caller-owned DEVICE memory (16-byte aligned), written by gaccum_ema_init and afterwards only
 * by the apply launches. */
typedef struct gaccum_ema_state {
  int64_t num_updates; /* n: windows averaged so far */
  float decay;         /* d of the last averaged window (0 before the first) */
  float reserved;
} gaccum_ema_state;

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
 * and `adam_m` / `adam_v` (optimization.py:137-148).  device = -1: layout-only plan.
 * Limits of the layout, each refused with GACCUM_EINVAL: a tensor holds at most 2^32 - 1 elements (a tile's offset
 * inside its tensor is 32-bit); the padded slab (gaccum_padded_size) holds at most 2^37 elements, 512 GB in fp32 (a
 * tile's slab offset is 32-bit in units of 32 elements); a plan has fewer than 2^31 tiles.  Element counts, offsets and
 * byte counts are int64 everywhere, and every kernel forms its addresses in 64 bits. */
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
/* Algorithmic bytes of one launch: accumulate = 12 B x P; apply = 36 B x P (SURVEY.md 8(d)).
 * The first accumulate of a window does not read the accumulators (8 B x P; see gaccum_step), so
 * a window of N >= 2 micro-steps moves (8 + 12 (N-2) + 36) B x P.  The plan does not know N: the
 * accumulate figure stays 12 B x P.  A 16-bit plan (gaccum_plan_set_param_dtype) reads 2-byte gradients:
 * accumulate = 10 B x P (first of a window 6 B x P); apply = 36 B x P (the 2 bytes saved on G are spent on
 * the model copy).  A GACCUM_LAMB apply moves 48 B x P (fp32 or 16-bit): those 36, plus p read a second time and the
 * update u written and read back (the a' round trip of a clipped or loss-scaled apply is not counted, as above).
 * A plan that keeps an EMA (gaccum_plan_set_ema) reads and writes the average on every apply: 8 B x P more (44, or
 * 56 for GACCUM_LAMB). */
GACCUM_API int64_t gaccum_algorithmic_bytes(const gaccum_plan* plan, int32_t is_apply);

/* Trains a bf16 or fp16 model (dtype GACCUM_DTYPE_BF16 / GACCUM_DTYPE_F16) with fp32 master weights.  Host-only:
 * validates its arguments and keeps `master_slab`, which must be a 16-byte aligned device slab of
 * gaccum_padded_size() floats in the plan's layout (gaccum_offsets), holding the fp32 weights (e.g. the exact upcast
 * of the model's).  Allowed only before the first compute call on the plan, like gaccum_plan_set_loss_scale; the two
 * combine in either order.  From then on gaccum_step, gaccum_accumulate and gaccum_apply read grads[i] and params[i]
 * as pointers to 16-bit tensors (any 2-byte alignment; 8-byte alignment takes the vector path).  The gradients are
 * widened exactly and accumulated in fp32; the apply updates the master weights exactly as an fp32 plan updates its
 * parameters, then stores params[i] = the master weights rounded to nearest-even (also after tensors without a
 * gradient; never on a window that loss scaling skips).  The master weights are the truth: params[i] is an output.
 * gaccum_step_packed, gaccum_step_dp, gaccum_apply_dp, gaccum_host_session_create and gaccum_step_host refuse such a
 * plan with GACCUM_EINVAL. */
GACCUM_API int gaccum_plan_set_param_dtype(gaccum_plan* plan, int32_t dtype, float* master_slab);

/* Turns dynamic loss scaling on for this plan (see gaccum_loss_scale_config).  Host-only: validates `cfg` and keeps
 * `device_state` (non-NULL, 16-byte aligned; not dereferenced here).  Allowed only before the first call of a compute
 * entry point on the plan (gaccum_step, _accumulate, _apply, _step_packed, _step_dp, _apply_dp), returns
 * GACCUM_EINVAL afterwards.  gaccum_step, gaccum_apply and gaccum_step_packed then apply with loss scaling, whatever
 * clip_norm is: their apply step is the two-pass clip-apply kernel (with clip_norm <= 0 it does not clip, but still
 * checks every element before it writes).  gaccum_accumulate is unchanged.  gaccum_step_dp, gaccum_apply_dp,
 * gaccum_host_session_create and gaccum_step_host refuse a loss-scaled plan with GACCUM_EINVAL. */
GACCUM_API int gaccum_plan_set_loss_scale(gaccum_plan* plan, const gaccum_loss_scale_config* cfg,
                                          gaccum_loss_scale_state* device_state);
/* GACCUM_LAMB: which tensors get layer adaptation (adapt[i] != 0: the update is scaled by the trust ratio; 0: r = 1).
 * Without a call every tensor adapts.  Allowed on LAMB plans only, and only before the first compute call on the plan,
 * like gaccum_plan_set_loss_scale; adapt[] (num_tensors bytes, host memory) is copied, synchronously into the plan's
 * device memory on a device plan. */
GACCUM_API int gaccum_plan_set_layer_adaptation(gaccum_plan* plan, const uint8_t* adapt);

/* Writes the initial state into `device_state` asynchronously on `stream`: scale = initial_scale, the three counters 0,
 * beta powers fp32(beta1) and fp32(beta2) (TF1's initial values).  The plan must have loss scaling on. */
GACCUM_API int gaccum_loss_scale_init(gaccum_plan* plan, gaccum_loss_scale_state* device_state, gaccum_stream_t stream);

/* Keeps an exponential moving average of the weights (see gaccum_ema_config).  Host-only: validates `cfg` and keeps
 * `ema_slab` (a 16-byte aligned device slab of gaccum_padded_size() floats in the plan's layout, holding the initial
 * averages) and `device_state` (16-byte aligned; not dereferenced here).  Allowed only before the first compute call on
 * the plan, like gaccum_plan_set_loss_scale; combines with gaccum_plan_set_param_dtype, gaccum_plan_set_loss_scale and
 * gaccum_plan_set_layer_adaptation in any order.  gaccum_step, gaccum_apply and gaccum_step_packed then update the
 * average in their apply step; gaccum_step_dp, gaccum_apply_dp, gaccum_host_session_create and gaccum_step_host refuse
 * such a plan with GACCUM_EINVAL. */
GACCUM_API int gaccum_plan_set_ema(gaccum_plan* plan, const gaccum_ema_config* cfg, float* ema_slab,
                                   gaccum_ema_state* device_state);
/* Writes num_updates = `num_updates` (>= 0; e.g. from a checkpoint) and decay = 0 into `device_state` asynchronously on
 * `stream`.  The plan must keep an EMA, and `device_state` must be the block given to gaccum_plan_set_ema (GACCUM_EINVAL
 * otherwise: the apply reads that one). */
GACCUM_API int gaccum_ema_init(gaccum_plan* plan, gaccum_ema_state* device_state, int64_t num_updates, gaccum_stream_t stream);

/* Per-tensor learning rates (layer-wise learning-rate decay, parameter groups): tensor t trains with
 *     lr_t = fp32(lr * mult[t])                 one correctly rounded fp32 multiply, as TF's `learning_rate * python_float`
 * in place of the step's lr, wherever the variant uses it:
 *     GACCUM_ADAM_WEIGHT_DECAY   p = p - lr_t*u                        (u includes the decay term, as in ELECTRA)
 *     GACCUM_ADAM                alpha_t = (lr_t * sqrt(1 - beta2_power)) / (1 - beta1_power), make_scalars' op order
 *                                (loss-scaled: the device block's beta powers)
 *     GACCUM_LAMB                p = p - (r*lr_t)*u
 * mult[t] is an fp32 value, finite and >= 0; 1.0 for every tensor without a call.  Nothing else depends on the
 * multipliers, bit for bit: the accumulators, the global norm, the clip scale, the trust ratios, the loss-scaling decision
 * and state, the beta powers, the EMA rule and the stats (gaccum_stats.lr stays the step's lr).  Since x * 1.0f == x, a
 * plan whose multipliers are all 1 computes exactly what a plan without the call computes; a tensor with multiplier 0
 * keeps its weights while its m and v advance.
 * `mult` is num_tensors floats in host memory, copied -- synchronously into the plan's device memory on a device plan.
 * GACCUM_EINVAL for NULL, a NaN, an infinity or a negative value, and after the plan's first compute call, like
 * gaccum_plan_set_loss_scale; combines with the other setters in any order.  gaccum_algorithmic_bytes is unchanged: the
 * num_tensors x 4-byte table is plan metadata, as the tile table is.  gaccum_step_dp, gaccum_apply_dp,
 * gaccum_host_session_create and gaccum_step_host refuse a plan on which it was called with GACCUM_EINVAL. */
GACCUM_API int gaccum_plan_set_lr_multipliers(gaccum_plan* plan, const float* mult);

/* Per-token normalisation of each accumulation window (token-level losses such as masked-LM pretraining).  Dividing
 * by N averages the micro-batches' mean losses; that equals the gradient of the large batch a window stands for only
 * when every micro-batch carries the same loss weight.  With this setter each window is divided by its total weight:
 *   - the producer differentiates the SUMMED loss of each micro-batch, and adds that micro-batch's weight w_i (its
 *     number of loss tokens, typically; any fp32 value) into `weight` with fp32 adds, on the device;
 *   - the apply step computes c = a' / W in place of (1.0 * a') / N.  If W is a normal power of two this is an exact
 *     multiply by 1/W, else a correctly rounded division -- the rule the unweighted apply uses for N -- so c is always
 *     the correctly rounded a' / W.  Everything after it is unchanged: * 1/S under loss scaling, the global norm and
 *     the clip scale (computed on c), every variant's update, the EMA, the learning-rate multipliers, the stats;
 *   - N still decides where a window ends (gaccum_is_apply_step); it no longer divides.  The reference divides the
 *     one-micro-batch window at global_step 0 by N; a weighted plan divides it by its own W;
 *   - every apply launch, applied or skipped by loss scaling, stores last_weight = W and resets weight = +0.
 *     Accumulate steps never touch the block;
 *   - the producer must have added ALL of the window's weights -- the apply step's own micro-batch included -- before
 *     the apply step is enqueued on the stream.  The total can arrive at the end of the window: nothing is read on the
 *     host, so the window can be captured in a CUDA graph together with the producer's adds.
 * A W that is not positive and finite is the caller's error.  The library reads no device data on the host, so IEEE
 * results propagate (W = 0 gives infinities and NaNs in c), as a NaN gradient propagates in the reference; with loss
 * scaling and clipping on, the non-finite global norm skips such a window.
 * `state` is caller-owned device memory, 16-byte aligned; zeroed memory is the starting state.  The setter is host-only
 * and reads nothing through the pointer.  GACCUM_EINVAL for NULL or a misaligned block, and after the plan's first
 * compute call; combines with the other setters in any order.  gaccum_step, gaccum_apply and gaccum_step_packed honour
 * it; gaccum_step_dp, gaccum_apply_dp, gaccum_host_session_create and gaccum_step_host refuse such a plan with
 * GACCUM_EINVAL.  gaccum_algorithmic_bytes is unchanged (the block is 16 bytes per window). */
typedef struct gaccum_window_weight_state {
  float weight;       /* W: the running window's total weight, added by the producer */
  float last_weight;  /* W of the last apply launch (written by the apply) */
  float reserved[2];
} gaccum_window_weight_state;
GACCUM_API int gaccum_plan_set_window_weight(gaccum_plan* plan, gaccum_window_weight_state* state);

/* The device schedule: global_step, the learning rate and TF1's beta powers kept on the device, so a CUDA graph of one
 * window of micro-steps (producer + train op) can be replayed for the whole run.  Off unless set; a plan without it
 * takes lr and the beta powers from gaccum_step_args, exactly as before.
 *   - The block (gaccum_schedule_state, caller-owned device memory) holds the step, the beta powers and the schedule
 *     constants; gaccum_schedule_init writes it, afterwards only the launches do.
 *   - Every launch of gaccum_step / gaccum_step_packed reads g = global_step, computes
 *         lr = gaccum_learning_rate(init_lr, num_train_steps, num_warmup_steps, g)
 *     with the same fp32 ops in the same order (bit for bit the host's lr; create_optimizer's polynomial decay with
 *     end_lr = 0 and power = 1, optimization.py:29-52), uses it wherever gaccum_step_args.lr would go (the per-tensor
 *     multipliers then apply as before, lr_t = fp32(lr * mult[t])), writes it to the stats, and stores
 *     global_step = g + 1 -- accumulate launches and windows that loss scaling skips included.
 *   - The beta powers have ONE home.  Without loss scaling it is this block: an applied window of GACCUM_ADAM or
 *     GACCUM_LAMB uses them, then multiplies each by fp32(beta) once (TF1 AdamOptimizer._finish).  Under loss scaling it
 *     is the loss-scaling block (gaccum_loss_scale_state.beta{1,2}_power), as without a device schedule; this block's
 *     beta fields are then 0 and unused.
 *   - The host still chooses the kernel, from gaccum_step_args.global_step and accum_n as before: the branch, and for an
 *     accumulate whether it is the window's first (which does not read the accumulators).  Eager launches should pass
 *     the step they run at.  Each launch checks g against its kernel: (int32)g % N == 0 exactly for an apply, and a
 *     first accumulate only where (int32)(g - 1) % N == 0.  A launch that finds otherwise changes nothing and sets
 *     `refused`; from then on every launch on the plan is a no-op, until gaccum_schedule_init rewrites the block.
 *     gaccum_step_args.lr and .beta{1,2}_power are ignored.
 *   - A graph captured over whole windows replays correctly at any g whose windows are N launches each (N - 1
 *     accumulates, the first without reading the accumulators, then an apply).  That holds for every g except across
 *     the int32 wrap: (int32)g jumps from 2^31 - 1 to -2^31 at g = 2^31 + k 2^32, and unless N is a power of two the
 *     window that straddles the jump is longer than N (N = 3: applies at 2^31 - 2, then 2^31 + 2).  A replay that
 *     reaches that window is refused at its first launch whose kernel g does not select, after the launches before it
 *     ran.  The caller then reads global_step, rewrites the block with gaccum_schedule_init at that step, runs the
 *     straddling window's remaining micro-steps eagerly (each with its own step), and replays again from the next
 *     window start.  A replay whose capture did not start at a window start, or did not end at a window end, is
 *     refused the same way.
 *   - gaccum_step_packed must use force_branch = -1; on an accumulate step its grad_slab may be NULL (the gradients
 *     are already in accum): the launch then only advances the schedule.
 * gaccum_plan_set_device_schedule is host-only: validates `cfg` (end_lr must be 0 and power 1) and keeps `block`
 * (16-byte aligned; not dereferenced here).  Allowed only before the plan's first compute call; combines with the other
 * setters in any order.  gaccum_accumulate and gaccum_apply (no step to check), gaccum_step_dp, gaccum_apply_dp,
 * gaccum_host_session_create and gaccum_step_host refuse such a plan with GACCUM_EINVAL. */
typedef struct gaccum_schedule_config {
  double init_lr;           /* optimization.py:29, rounded to fp32 as the host schedule does */
  int64_t num_train_steps;  /* >= 0 */
  int64_t num_warmup_steps; /* >= 0; 0: no warm-up */
  double end_lr;            /* must be 0 */
  double power;             /* must be 1 */
} gaccum_schedule_config;
typedef struct gaccum_schedule_state {
  int64_t global_step;      /* the pre-increment step of the next launch */
  int64_t num_train_steps;
  int64_t num_warmup_steps;
  float init_lr;            /* fp32(init_lr) */
  float end_lr;             /* 0 */
  float power;              /* 1 */
  float beta1_power;        /* without loss scaling: TF1's beta1^t (see above) */
  float beta2_power;
  int32_t refused;          /* 1 once a launch found global_step selecting the other branch */
} gaccum_schedule_state;    /* 48 bytes */
GACCUM_API int gaccum_plan_set_device_schedule(gaccum_plan* plan, const gaccum_schedule_config* cfg,
                                               gaccum_schedule_state* block);
/* Writes the block on `stream` (stream-ordered; the call returns once the host values are staged): global_step,
 * beta{1,2}_power (ignored under loss scaling: they live in the loss-scaling block), the plan's schedule constants and
 * refused = 0.  `block` must be the one given to gaccum_plan_set_device_schedule. */
GACCUM_API int gaccum_schedule_init(gaccum_plan* plan, gaccum_schedule_state* block, int64_t global_step,
                                    float beta1_power, float beta2_power, gaccum_stream_t stream);

/* A learning-rate table for the device schedule, so a replayed CUDA graph follows any schedule the host can evaluate
 * (polynomial decay with any power and end value, cosine, exponential, piecewise-constant, each with or without BERT's
 * warm-up): the host evaluates it once per step, the device looks it up.
 *   - Every launch of a table plan (gaccum_step, gaccum_step_packed, accumulates included) uses
 *         lr = device_table[min(g, length - 1)]
 *     in place of gaccum_learning_rate(init_lr, num_train_steps, num_warmup_steps, g); g is the block's int64
 *     global_step (>= 0), so the index does not wrap with the int32 branch predicate.  That lr goes everywhere the
 *     formula's goes: lr_t = fp32(lr * mult[t]), GACCUM_ADAM's alpha, GACCUM_LAMB's r*lr_t and gaccum_stats.lr.
 *   - Nothing else changes: the branch predicate, `refused`, the beta powers, loss scaling, the moving average, the
 *     window weight, the per-tensor norms and 16-bit models behave as on any device-scheduled plan.  A table holding
 *     gaccum_learning_rate(g) at every g computes exactly what the formula computes.
 *   - The table is read at launch time, stream-ordered: a caller may rewrite entries between launches or graph replays
 *     and the next launch that reads an entry uses its new value.  Non-finite or negative entries are the caller's
 *     error: IEEE results propagate, as with a NaN gradient.
 * The plan must be device-scheduled (gaccum_plan_set_device_schedule, whose cfg is still validated; the table then
 * ignores its init_lr, num_train_steps and num_warmup_steps).  The setter is host-only: `device_table` is caller-owned
 * device memory of `length` >= 1 floats, 4-byte aligned, not dereferenced here and read by every launch after it.
 * Allowed only before the plan's first compute call; combines with the other setters in any order; a first compute call
 * on a plan that has a table but no device schedule fails with GACCUM_EINVAL.  GACCUM_EINVAL for a NULL plan or table,
 * length < 1, a misaligned table, a layout-only plan, and after the first compute call.  gaccum_accumulate,
 * gaccum_apply, gaccum_step_dp, gaccum_apply_dp, gaccum_host_session_create and gaccum_step_host refuse a table plan
 * with GACCUM_EINVAL.  gaccum_algorithmic_bytes is unchanged (one 4-byte load per CTA). */
GACCUM_API int gaccum_plan_set_lr_table(gaccum_plan* plan, const float* device_table, int64_t length);

/* Per-tensor norms of the apply step, for watching a run layer by layer (TF1's add_gradients_summaries /
 * optimize_loss(summaries=["gradient_norm"])) without extra passes over the slabs.  Off unless set.  Every apply launch
 * of gaccum_step, gaccum_apply (grads == NULL included) and gaccum_step_packed writes, for every tensor t, row t of
 * `device_out` (num_tensors x 3 floats, caller-owned device memory, 16-byte aligned):
 *     [3t + 0]  gradient  ||c_t||: c the window gradient the update consumes BEFORE the clip scale -- (1.0 * a') / N (or
 *                         a' / W with a window weight), times 1/S under loss scaling: the c whose norm
 *                         gaccum_stats.global_norm reports -- whether clipping is on or off.  A tensor without a gradient
 *                         this micro-step reports the norm of its accumulated c.
 *     [3t + 1]  weight    ||p_t|| of the weights before the update (a 16-bit plan: the fp32 master weights).
 *     [3t + 2]  update    ||p_before - p_after||, from the per-element fp32 difference of what the apply stored: 0 for a
 *                         tensor with learning-rate multiplier 0, and 0 everywhere on a window that loss scaling skips.
 *   ||x|| = sqrtf(fp32(sum x^2)).  Each thread of the kernel sums x^2 of its elements of a tile in fp32 (fmaf, as the
 *   global norm's partials), a warp adds its threads' sums in fp64 in a fixed butterfly order, and those fp64 values are
 *   added tile by tile, warp by warp in a fixed order that depends on the tile table only: the values are bit-identical
 *   from launch to launch, across CUDA-graph replays and whichever CTA took a tile.  Non-finite values propagate (a
 *   tensor holding an inf reports inf, one holding a NaN reports NaN); a zero-element tensor reports 0.
 *   A window that loss scaling skips still writes all three columns: the overflowed tensors' gradient norms, the
 *   unchanged weights' norms and zero update norms.  Every apply launch overwrites the values; after a replayed graph of
 *   k windows they hold the last window's, as the stats block does.
 * Nothing else the apply computes depends on the setting, bit for bit.  The setter is host-only: it validates its
 * arguments, allocates the plan's scratch (per tile 192 bytes of fp64 partials, per 32 tiles 24 bytes, 12 bytes per
 * tensor of tables and counters) and zeroes `device_out` and waits for that to finish, so the values are 0 before the first apply.
 * GACCUM_EINVAL for a NULL plan or buffer, a misaligned buffer, a layout-only plan, and after the plan's first compute
 * call; combines with the other setters in any order.  gaccum_accumulate is unaffected; gaccum_step_dp,
 * gaccum_apply_dp, gaccum_host_session_create and gaccum_step_host refuse such a plan with GACCUM_EINVAL.
 * gaccum_algorithmic_bytes is unchanged: the scratch is metadata-sized. */
GACCUM_API int gaccum_plan_set_tensor_norms(gaccum_plan* plan, float* device_out);

/* ---- the hot path --------------------------------------------------------------------- */
/* One micro-step of the train_op (optimization.py:91-94): if gaccum_is_apply_step() the apply
 * branch (assign_add -> /N -> clip_by_global_norm -> apply_gradients -> zero; :80-88), else
 * the accumulate branch (:93).  grads[i] / params[i]: device pointers to tensor i (scattered,
 * any 4-byte alignment; 16-byte alignment takes the vector path).  grads[i] == NULL means
 * "no gradient for this tensor" (optimization.py:132 skips such pairs).  On a 16-bit plan
 * (gaccum_plan_set_param_dtype) grads[i] and params[i] point at bf16 / fp16 tensors, cast to float*.
 * accum / m / v: device slabs of gaccum_padded_size() floats, 16-byte aligned.
 * The caller increments global_step afterwards (optimization.py:102-103).
 * PRECONDITION, first micro-step of a window (global_step - 1 applies, global_step does not; never
 * at global_step 0 or with accum_n = 1): `accum` is not read and must hold +0.0 in every tensor
 * element; anything else there is overwritten, not added to.  That step stores accum = +0.0 + G
 * (tensors without a gradient keep their +0.0), which is what the reference computes there: its
 * accumulators start as zeros (optimization.py:78) and every apply zeroes them (:86-87).  A zero-
 * initialised slab and the apply branch of this library leave exactly that; a caller that writes
 * `accum` itself (e.g. restoring a checkpoint) must not leave non-zero values at a window start.
 * The same holds for gaccum_step_packed with force_branch = -1, gaccum_step_dp and gaccum_step_host.
 * gaccum_accumulate, and gaccum_step_packed with a forced branch, always compute accum += G. */
GACCUM_API int gaccum_step(gaccum_plan* plan, const float* const* grads, float* const* params,
                           float* accum, float* m, float* v, const gaccum_step_args* args,
                           gaccum_stream_t stream);
/* Deferred reset of the accumulators, as zero_grad(set_to_none=True) defers a gradient's reset: off unless set.  The
 * apply branch then stores nothing into `accum` (32 instead of 36 B x P, with clipping also no write-back of a' lines
 * still in L2) and leaves the accumulators LOGICALLY +0.0 on applied and loss-scale-skipped windows alike, for every
 * optimizer: a plan-owned device word records it and the slab's contents are unspecified until the next write.  The
 * first micro-step of a window (the precondition above) stores +0.0 + G where there is a gradient and, while the word
 * is set, +0.0 where there is none, then clears the word; its results are bit for bit those of a plan without the mode.
 * Every other launch that READS accum -- gaccum_accumulate, gaccum_apply, a gaccum_step that is not a window's first
 * accumulate, and any read or write of the slab by the caller -- must follow gaccum_accum_materialize on the same stream
 * when an apply may have run since the last first accumulate (e.g. after global_step was reassigned).
 *   gaccum_plan_set_deferred_reset: on = 1 or 0; host-only, at any time.  Turning the mode off does not write the slab:
 *   materialize first.  GACCUM_EINVAL for a NULL or layout-only plan, or on not 0 or 1.  gaccum_step_dp,
 *   gaccum_apply_dp, gaccum_host_session_create and gaccum_step_host refuse such a plan with GACCUM_EINVAL.
 *   gaccum_step_packed ignores the mode (its caller adds into the slab between launches, so the slab holds real zeros):
 *   its applies store them and it neither reads nor writes the word -- a slab it shares with launches of the mode is
 *   materialized first.  gaccum_algorithmic_bytes is unchanged.
 *   gaccum_accum_materialize: asynchronous on `stream` and graph-capturable; stores +0.0 into every tensor element of
 *   `accum` if the word is set (4 B x P) and clears it, else changes nothing; it reads and writes no other device state
 *   (not gaccum_stats, the device schedule or any other block).  GACCUM_OK without a launch on a plan without the mode. */
GACCUM_API int gaccum_plan_set_deferred_reset(gaccum_plan* plan, int32_t on);
GACCUM_API int gaccum_accum_materialize(gaccum_plan* plan, float* accum, gaccum_stream_t stream);
/* The two branches on their own (the data-parallel driver accumulates locally, all-reduces the
 * slab, then applies with grads == NULL).  gaccum_apply ignores args->global_step.
 * gaccum_accumulate has no step arguments and always reads accum: accum += G for any accum.
 * On a 16-bit plan both take 16-bit grads[i] / params[i], as gaccum_step does. */
GACCUM_API int gaccum_accumulate(gaccum_plan* plan, const float* const* grads, float* accum,
                                 gaccum_stream_t stream);
GACCUM_API int gaccum_apply(gaccum_plan* plan, const float* const* grads, float* const* params,
                            float* accum, float* m, float* v, const gaccum_step_args* args,
                            gaccum_stream_t stream);
/* Same step when gradients and parameters are themselves packed in slab layout (params as
 * views of one flat buffer): no pointer table.  grad_slab may be NULL on an apply step.
 * With force_branch = -1 the first micro-step of a window has gaccum_step's precondition; a forced
 * accumulate (force_branch = 0) cannot know what the previous micro-step did and reads accum. */
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
 * On the first micro-step of a window comm->accum is not read and must hold +0.0 (gaccum_step's
 * precondition); the apply step leaves every rank's accumulators there.
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
 * parameters on apply steps.  stats_out (may be NULL) receives the stats block every step.
 * The session's accumulators start zeroed and its apply steps zero them, so gaccum_step's
 * precondition on the first micro-step of a window holds unless the caller writes them through
 * gaccum_host_session_slabs. */
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
/* GACCUM_LAMB: asynchronously copy the trust ratios r of the last applied window (num_tensors floats; 1 for tensors
 * without layer adaptation, and everywhere before the first applied window) to host memory, like gaccum_read_stats.  A
 * window that loss scaling skips leaves them.  GACCUM_EINVAL on other variants, GACCUM_ENODEVICE on a layout-only plan. */
GACCUM_API int gaccum_read_trust_ratios(gaccum_plan* plan, float* host_out, gaccum_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* GACCUM_H_ */
