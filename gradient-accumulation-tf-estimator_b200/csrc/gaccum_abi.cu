// gaccum_abi.cu -- host side of libgaccum.so: plan (slab layout + static tile table), the
// scalar host logic of the reference graph, and the C ABI declared in include/gaccum.h.
// No CPU compute path exists here on purpose: without a device every step call fails.
#include <regex.h>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <new>
#include <string>
#include <vector>

#include "../../include/gaccum.h"
#include "gaccum_kernels.cuh"
#include "gaccum_dp.cuh"
#include "gaccum_lamb.cuh"

using namespace gaccum;

// ------------------------------------------------------------------------------------------
// errors
// ------------------------------------------------------------------------------------------
static thread_local std::string g_err;

static int fail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  g_err = buf;
  return code;
}
#define CUDA_TRY(expr)                                                                        \
  do {                                                                                        \
    cudaError_t e_ = (expr);                                                                  \
    if (e_ != cudaSuccess)                                                                    \
      return fail(GACCUM_ECUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e_), __FILE__, __LINE__); \
  } while (0)

// ------------------------------------------------------------------------------------------
// plan
// ------------------------------------------------------------------------------------------
constexpr int kCapSmall = 256;    // 4 KB pointer table   (MNIST, BERT-Small 73, BERT-Base 201)
constexpr int kCapLarge = 1920;   // 30 KB pointer table  (BERT-Large 393, ...; CUDA >= 12.1 32 KB params)

struct gaccum_plan {
  int32_t T = 0;
  int32_t device = -1;
  gaccum_hparams hp{};
  std::vector<int64_t> numel, offset;
  std::vector<uint8_t> decay;
  std::vector<TileDesc> tiles;
  int64_t P = 0, padded = 0;
  // device side
  TileDesc* d_tiles = nullptr;
  double* d_partials = nullptr;            // data-parallel apply: one fp64 norm partial per block
  float* d_stats = nullptr;
  uint32_t* d_dp_sync = nullptr;           // data-parallel kernel: block-completion counters and tile tickets (zero between launches)
  unsigned long long* d_barrier = nullptr; // clip-apply kernel: monotonic arrival counter of the consumers' grid barrier
  LaunchCounters* d_counters = nullptr;    // ... two sets of per-launch counters (tickets, pool length, norm accumulator)
  unsigned int* d_done = nullptr;          // apply_kernel, scheduled accumulate_kernel: CTAs of the launch that are through (zero between launches)
#ifdef GACCUM_EXPERIMENTS
  unsigned long long* d_debug = nullptr;   // per-CTA timestamps (tools/cta_timeline.py; experiments build only)
#endif
  int num_sms = 0;
  int max_grid = 0;
  // dynamic loss scaling (gaccum_plan_set_loss_scale); may be turned on only while `computed` is false
  bool computed = false;
  bool ls_on = false;
  gaccum_loss_scale_config ls_cfg{};
  gaccum_loss_scale_state* ls_state = nullptr;
  // 16-bit model (gaccum_plan_set_param_dtype); set only while `computed` is false
  int32_t param_dtype = GACCUM_DTYPE_F32;
  float* master = nullptr;
  // GACCUM_LAMB: per-tensor layer-adaptation flags (gaccum_plan_set_layer_adaptation), the exact per-tensor norm
  // accumulators (two sets) and the trust ratios of the last applied window
  std::vector<uint8_t> adapt;
  uint8_t* d_adapt = nullptr;
  LambTensorAcc* d_lamb_acc = nullptr;
  float* d_ratios = nullptr;
  // exponential moving average of the weights (gaccum_plan_set_ema); set only while `computed` is false
  bool ema_on = false;
  gaccum_ema_config ema_cfg{};
  float* ema_slab = nullptr;
  gaccum_ema_state* ema_state = nullptr;
  // per-tensor learning-rate multipliers (gaccum_plan_set_lr_multipliers): 1.0 unless set, the device copy exists on every
  // device plan because every apply kernel reads it
  bool lr_mult_set = false;
  std::vector<float> lr_mult;
  float* d_lr_mult = nullptr;
  // per-window normalisation by the producer's total weight (gaccum_plan_set_window_weight); set only while `computed`
  // is false
  gaccum_window_weight_state* ww_state = nullptr;
  // the device schedule (gaccum_plan_set_device_schedule); set only while `computed` is false
  gaccum_schedule_config sched_cfg{};
  gaccum_schedule_state* sched_state = nullptr;
  // a learning-rate table of the device schedule (gaccum_plan_set_lr_table); set only while `computed` is false
  LrTableParams lr_table{};
  // per-tensor norms of the apply step (gaccum_plan_set_tensor_norms); set only while `computed` is false.  d_norms holds
  // the partials, the chunk tables and the counters of NormParams in one allocation
  NormParams norms{};
  void* d_norms = nullptr;
  // deferred reset of the accumulators (gaccum_plan_set_deferred_reset): d_reset holds the word accum_zero (unsigned int
  // 0) and, at floats 4 .. 7, the stats block gaccum_accum_materialize's launch writes instead of gaccum_stats
  bool deferred = false;
  unsigned int* d_reset = nullptr;
  std::mutex mu;
  std::map<const void*, int> grid_cache;   // cooperative kernel -> CTAs that fit on one SM (fit)
};

static int build_layout(gaccum_plan* pl) {
  pl->offset.resize(pl->T);
  int64_t off = 0, P = 0;
  pl->tiles.clear();
  for (int32_t t = 0; t < pl->T; ++t) {
    const int64_t n = pl->numel[t];
    if (n < 0) return fail(GACCUM_EINVAL, "numels[%d] = %lld is negative", t, (long long)n);
    if (n >= (int64_t)1 << 32) return fail(GACCUM_EINVAL, "tensor %d has %lld elements; limit is 2^32-1", t, (long long)n);
    // the padded slab ends at or before 2^37, so every tile's slab offset / kSlabAlign fits TileDesc::soff32
    const int64_t padded_n = (n + kSlabAlign - 1) / kSlabAlign * kSlabAlign;
    if (off + padded_n > (int64_t)1 << 37) return fail(GACCUM_EINVAL, "slab too large (> 2^37 elements)");
    pl->offset[t] = off;
    for (int64_t to = 0; to < n; to += kTile) {
      TileDesc d;
      d.tensor_flags = (uint32_t)t | (pl->decay[t] ? 0x80000000u : 0u);
      d.len = (uint32_t)std::min<int64_t>(kTile, n - to);
      d.toff = (uint32_t)to;
      d.soff32 = (uint32_t)((off + to) / kSlabAlign);
      pl->tiles.push_back(d);
    }
    P += n;
    off += padded_n;
  }
  if (pl->tiles.size() >= (size_t)1 << 31) return fail(GACCUM_EINVAL, "too many tiles");
  pl->P = P;
  pl->padded = off;
  return GACCUM_OK;
}

// ------------------------------------------------------------------------------------------
// scalars of one apply step
// ------------------------------------------------------------------------------------------
static Scalars make_scalars(const gaccum_hparams& hp, const gaccum_step_args* a) {
  Scalars s{};
  s.nf = a ? (float)a->accum_n : 1.0f;
  {
    const int32_t n = a ? a->accum_n : 1;
    s.inv_nf = (n > 0 && (n & (n - 1)) == 0 && n <= (1 << 24)) ? 1.0f / (float)n : 0.0f;
  }
  s.lr = a ? a->lr : 0.0f;
  s.b1p = a ? a->beta1_power : 0.0f;
  s.b2p = a ? a->beta2_power : 0.0f;
  s.b1 = (float)hp.beta1;
  s.b2 = (float)hp.beta2;
  s.eps = (float)hp.epsilon;
  s.wd = (float)hp.weight_decay_rate;
  s.clip = (float)hp.clip_norm;
  if (hp.variant != GACCUM_ADAM) {
    s.omb1 = (float)(1.0 - hp.beta1);   // optimization.py:152 -- Python double, then fp32 (GACCUM_LAMB the same)
    s.omb2 = (float)(1.0 - hp.beta2);   // optimization.py:154
  } else {
    volatile float o1 = 1.0f - s.b1, o2 = 1.0f - s.b2;   // ApplyAdam: T(1) - beta1()
    s.omb1 = o1;
    s.omb2 = o2;
  }
  return s;
}

// ------------------------------------------------------------------------------------------
// launch helpers
// ------------------------------------------------------------------------------------------
// The CTAs of `threads` threads and `smem` bytes of dynamic shared memory that fit on one SM, found once per kernel
// (which also sets the kernel's dynamic shared memory limit).  A cooperative kernel's grid must be co-resident, and the
// grid of the clip-apply and LAMB kernels depends on the plan alone (their barrier counter advances by gridDim.x), so a
// kernel that fits fewer than `need` CTAs per SM is an error, never a smaller grid.
static int fit(gaccum_plan* pl, const void* fn, const char* name, int threads, int smem, int need, int* per_sm) {
  std::lock_guard<std::mutex> lk(pl->mu);
  auto it = pl->grid_cache.find(fn);
  if (it == pl->grid_cache.end()) {
    if (smem > 0) CUDA_TRY(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    int n = 0;
    CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, fn, threads, (size_t)smem));
    if (n < need) {
      return need == 1 ? fail(GACCUM_ECUDA, "%s does not fit on an SM (%d B dynamic shared memory)", name, smem)
                       : fail(GACCUM_ECUDA, "%s fits %d CTAs per SM, it needs %d", name, n, need);
    }
    it = pl->grid_cache.emplace(fn, n).first;
  }
  *per_sm = it->second;
  return GACCUM_OK;
}

// from_zero: the accumulators hold +0.0 (first micro-step of a window), so the kernel does not read them
// H: a 16-bit model (gaccum_plan_set_param_dtype), scattered pointer tables only
template <int CAP, bool H = false>
static int launch_accumulate(gaccum_plan* pl, KernelParams<CAP>& prm, bool from_zero, cudaStream_t st) {
  // one tile per CTA: the hardware block scheduler balances better than a persistent loop
  const int grid = std::max(1, prm.num_tiles);
  if (from_zero) accumulate_kernel<CAP, true, H><<<grid, kThreads, 0, st>>>(prm);
  else accumulate_kernel<CAP, false, H><<<grid, kThreads, 0, st>>>(prm);
  CUDA_TRY(cudaGetLastError());
  return GACCUM_OK;
}

// The apply step: the kernel of the plan's (variant, mode) and its launch shape.  Loss scaling always takes a
// cooperative kernel: the single-pass apply_kernel stores p, m and v before it could know whether the window overflowed.
//   apply_kernel       AdamWeightDecay / Adam in kNoClip: one tile per CTA
//   apply_clip_kernel  AdamWeightDecay / Adam in every other mode: ONE 864-thread CTA per SM (ring + stash take nearly
//                      all of the SM's shared memory, so a second CTA could never be co-resident), min(SMs, ceil(nt/3))
//   lamb_apply_kernel  LAMB in every mode: kLambBlocksPerSm CTAs per SM, min(kLambBlocksPerSm x SMs, nt)
template <int CAP, bool H, bool EMA>
static int launch_apply(gaccum_plan* pl, KernelParams<CAP>& prm, cudaStream_t st) {
  const bool clip = pl->hp.clip_norm > 0.0;
  const int mode = pl->ls_on ? (clip ? kLsClip : kLsNoClip) : (clip ? kClip : kNoClip);
  const int nt = (int)pl->tiles.size();
  const bool adam = pl->hp.variant == GACCUM_ADAM;
  if (pl->hp.variant != GACCUM_LAMB && mode == kNoClip) {
    if (adam) apply_kernel<1, CAP, H, EMA><<<std::max(1, nt), kThreads, 0, st>>>(prm);
    else apply_kernel<0, CAP, H, EMA><<<std::max(1, nt), kThreads, 0, st>>>(prm);
    CUDA_TRY(cudaGetLastError());
    return GACCUM_OK;
  }
  static_assert(kNoClip == 0 && kClip == 1 && kLsClip == 2 && kLsNoClip == 3, "the tables are indexed by mode");
  static const void* const lamb[4] = {
      (const void*)&lamb_apply_kernel<CAP, kNoClip, H, EMA>, (const void*)&lamb_apply_kernel<CAP, kClip, H, EMA>,
      (const void*)&lamb_apply_kernel<CAP, kLsClip, H, EMA>, (const void*)&lamb_apply_kernel<CAP, kLsNoClip, H, EMA>};
  static const void* const clip_apply[2][4] = {   // [VARIANT][mode]
      {nullptr, (const void*)&apply_clip_kernel<0, CAP, kClip, H, EMA>, (const void*)&apply_clip_kernel<0, CAP, kLsClip, H, EMA>,
       (const void*)&apply_clip_kernel<0, CAP, kLsNoClip, H, EMA>},
      {nullptr, (const void*)&apply_clip_kernel<1, CAP, kClip, H, EMA>, (const void*)&apply_clip_kernel<1, CAP, kLsClip, H, EMA>,
       (const void*)&apply_clip_kernel<1, CAP, kLsNoClip, H, EMA>}};
  const bool is_lamb = pl->hp.variant == GACCUM_LAMB;
  const void* fn = is_lamb ? lamb[mode] : clip_apply[adam ? 1 : 0][mode];
  const int threads = is_lamb ? kThreads : kClipThreads;
  const int smem = is_lamb ? 0 : kClipSmemBytes;
  int per_sm = 0;
  if (int rc = fit(pl, fn, is_lamb ? "lamb_apply_kernel" : "apply_clip_kernel", threads, smem, is_lamb ? kLambBlocksPerSm : 1, &per_sm))
    return rc;
  const int grid = is_lamb ? std::max(1, std::min(pl->num_sms * kLambBlocksPerSm, nt))
                           : std::max(1, std::min(pl->num_sms, (nt + kGroups - 1) / kGroups));
  void* args[] = {(void*)&prm};
  CUDA_TRY(cudaLaunchCooperativeKernel(fn, dim3(grid), dim3(threads), args, (size_t)smem, st));
  return GACCUM_OK;
}

static inline bool aligned16_host(const void* p) { return ((uintptr_t)p & 15u) == 0; }

static int check_compute(gaccum_plan* pl, const float* accum, const float* m, const float* v, bool need_mv) {
  if (!pl) return fail(GACCUM_EINVAL, "plan is NULL");
  pl->computed = true;   // from here on gaccum_plan_set_loss_scale is refused
  if (pl->device < 0)
    return fail(GACCUM_ENODEVICE, "layout-only plan (device=-1): libgaccum has no CPU fallback, a CUDA device is required");
  if (pl->lr_table.table && !pl->sched_state)
    return fail(GACCUM_EINVAL, "a learning-rate table (gaccum_plan_set_lr_table) needs a device schedule "
                               "(gaccum_plan_set_device_schedule), which this plan lacks");
  if (!accum || !aligned16_host(accum)) return fail(GACCUM_EINVAL, "accum must be a 16-byte aligned device pointer");
  if (need_mv && (!m || !v || !aligned16_host(m) || !aligned16_host(v)))
    return fail(GACCUM_EINVAL, "m and v must be 16-byte aligned device pointers");
  return GACCUM_OK;
}

template <int CAP>
static void fill_common(gaccum_plan* pl, KernelParams<CAP>& prm, float* accum, float* m, float* v,
                        const gaccum_step_args* a) {
  prm.tiles = pl->d_tiles;
  prm.num_tiles = (int32_t)pl->tiles.size();
  prm.accum = accum;
  prm.m = m;
  prm.v = v;
  prm.barrier = pl->d_barrier;
  prm.counters = pl->d_counters;
  prm.done = pl->d_done;
#ifdef GACCUM_EXPERIMENTS
  prm.debug = pl->d_debug;
#endif
  prm.stats = pl->d_stats;
  prm.sc = make_scalars(pl->hp, a);
  if (pl->ls_on) {
    prm.ls.state = reinterpret_cast<LossScaleState*>(pl->ls_state);
    prm.ls.multiplier = (float)pl->ls_cfg.multiplier;
    prm.ls.growth_interval = pl->ls_cfg.growth_interval;
  }
  prm.half.master = pl->master;
  prm.half.bf16 = pl->param_dtype == GACCUM_DTYPE_BF16;
  prm.lamb.acc = pl->d_lamb_acc;
  prm.lamb.ratios = pl->d_ratios;
  prm.lamb.adapt = pl->d_adapt;
  prm.lamb.num_tensors = pl->T;
  prm.ema.slab = pl->ema_slab;
  prm.ema.state = reinterpret_cast<EmaState*>(pl->ema_state);
  prm.ema.decay = (float)pl->ema_cfg.decay;
  prm.ema.num_updates = pl->ema_cfg.num_updates;
  prm.lrm.mult = pl->d_lr_mult;
  prm.ww.state = reinterpret_cast<WindowWeightState*>(pl->ww_state);
  prm.sched.state = reinterpret_cast<ScheduleState*>(pl->sched_state);
  prm.sched.accum_n = a ? a->accum_n : 1;
  prm.norms = pl->norms;
  prm.lrt = pl->lr_table;
  prm.dr.accum_zero = pl->deferred ? pl->d_reset : nullptr;
}

template <int CAP>
static int fill_table(gaccum_plan* pl, PtrTable<CAP>& tab, const float* const* grads, float* const* params) {
  for (int32_t t = 0; t < pl->T; ++t) {
    tab.g[t] = grads ? grads[t] : nullptr;
    if (params) {
      if (!params[t] && pl->numel[t] > 0) return fail(GACCUM_EINVAL, "params[%d] is NULL", t);
      tab.p[t] = params[t];
    }
  }
  return GACCUM_OK;
}

struct DeviceGuard {
  int prev = -1;
  bool ok = false;
  explicit DeviceGuard(int dev) {
    if (cudaGetDevice(&prev) == cudaSuccess && prev != dev) ok = cudaSetDevice(dev) == cudaSuccess;
    else prev = -1;
  }
  ~DeviceGuard() { if (prev >= 0 && ok) cudaSetDevice(prev); }
};

// An accumulate step is the first of its window when the previous micro-step took the apply branch, which left every
// accumulator at +0.0 (optimization.py:86-87; they start as zeros, :78).  Both predicates take the reference's int32
// cast of the step; subtracting after the cast cannot overflow and wraps like the reference's int32 step would.
// False without step arguments (gaccum_accumulate), at global_step 0, and always for N = 1 (every step applies).
static bool first_of_window(const gaccum_step_args* a) {
  if (!a) return false;
  const int64_t prev = (int64_t)(int32_t)a->global_step - 1;
  return !gaccum_is_apply_step(a->global_step, a->accum_n) && gaccum_is_apply_step(prev, a->accum_n);
}

template <int CAP>
static int do_accumulate_tab(gaccum_plan* pl, const float* const* grads, float* accum,
                             const gaccum_step_args* a, cudaStream_t st) {
  KernelParams<CAP>* prm = new (std::nothrow) KernelParams<CAP>();
  if (!prm) return fail(GACCUM_ENOMEM, "out of host memory");
  fill_common(pl, *prm, accum, nullptr, nullptr, a);
  int rc = fill_table(pl, prm->tab, grads, nullptr);
  if (rc == GACCUM_OK) {
    rc = pl->master ? launch_accumulate<CAP, true>(pl, *prm, first_of_window(a), st)
                    : launch_accumulate<CAP, false>(pl, *prm, first_of_window(a), st);
  }
  delete prm;
  return rc;
}

template <int CAP>
static int do_apply_tab(gaccum_plan* pl, const float* const* grads, float* const* params, float* accum,
                        float* m, float* v, const gaccum_step_args* a, cudaStream_t st) {
  KernelParams<CAP>* prm = new (std::nothrow) KernelParams<CAP>();
  if (!prm) return fail(GACCUM_ENOMEM, "out of host memory");
  fill_common(pl, *prm, accum, m, v, a);
  int rc = fill_table(pl, prm->tab, grads, params);
  if (rc == GACCUM_OK) {
    if (pl->master) rc = pl->ema_on ? launch_apply<CAP, true, true>(pl, *prm, st) : launch_apply<CAP, true, false>(pl, *prm, st);
    else rc = pl->ema_on ? launch_apply<CAP, false, true>(pl, *prm, st) : launch_apply<CAP, false, false>(pl, *prm, st);
  }
  delete prm;
  return rc;
}

static int check_args(const gaccum_step_args* a) {
  if (!a) return fail(GACCUM_EINVAL, "args is NULL");
  if (a->accum_n <= 0) return fail(GACCUM_EINVAL, "accum_n must be > 0 (got %d)", a->accum_n);
  if (a->reserved != 0 || a->reserved2 != 0.0f) return fail(GACCUM_EINVAL, "reserved fields must be 0");
  return GACCUM_OK;
}

// The plan settings an entry point may lack (refuse), in the order refuse checks them
enum PlanSetting : unsigned {
  kPlanLossScale = 1u << 0,
  kPlanLamb = 1u << 1,
  kPlanHalf = 1u << 2,
  kPlanEma = 1u << 3,
  kPlanLrMult = 1u << 4,
  kPlanWindowWeight = 1u << 5,
  kPlanSchedule = 1u << 6,
  kPlanLrTable = 1u << 7,
  kPlanNorms = 1u << 8,
  kPlanDeferredReset = 1u << 9,
  kPlanAll = (1u << 10) - 1u,
};
// Fails on the first of the settings `lacks` names that the plan has: `what` does not support it
static int refuse(const gaccum_plan* pl, const unsigned lacks, const char* what) {
  if (!pl) return GACCUM_OK;
  const struct { unsigned setting; bool on; const char* name; } settings[] = {
      {kPlanLossScale, pl->ls_on, "loss scaling"},
      {kPlanLamb, pl->hp.variant == GACCUM_LAMB, "GACCUM_LAMB"},
      {kPlanHalf, pl->master != nullptr, "16-bit parameters (gaccum_plan_set_param_dtype)"},
      {kPlanEma, pl->ema_on, "a moving average (gaccum_plan_set_ema)"},
      {kPlanLrMult, pl->lr_mult_set, "learning-rate multipliers (gaccum_plan_set_lr_multipliers)"},
      {kPlanWindowWeight, pl->ww_state != nullptr, "a window weight (gaccum_plan_set_window_weight)"},
      {kPlanSchedule, pl->sched_state != nullptr, "a device schedule (gaccum_plan_set_device_schedule)"},
      {kPlanLrTable, pl->lr_table.table != nullptr, "a learning-rate table (gaccum_plan_set_lr_table)"},
      {kPlanNorms, pl->norms.out != nullptr, "per-tensor norms (gaccum_plan_set_tensor_norms)"},
      {kPlanDeferredReset, pl->deferred, "a deferred reset of the accumulators (gaccum_plan_set_deferred_reset)"},
  };
  for (const auto& st : settings)
    if ((lacks & st.setting) && st.on) return fail(GACCUM_EINVAL, "%s does not support %s", what, st.name);
  return GACCUM_OK;
}

static void free_plan_device(gaccum_plan* pl) {
  cudaFree(pl->d_tiles); cudaFree(pl->d_partials); cudaFree(pl->d_stats); cudaFree(pl->d_dp_sync); cudaFree(pl->d_barrier); cudaFree(pl->d_counters);
  cudaFree(pl->d_adapt); cudaFree(pl->d_lamb_acc); cudaFree(pl->d_ratios); cudaFree(pl->d_done); cudaFree(pl->d_lr_mult);
  cudaFree(pl->d_norms); cudaFree(pl->d_reset);
#ifdef GACCUM_EXPERIMENTS
  cudaFree(pl->d_debug);
#endif
}

// ------------------------------------------------------------------------------------------
// C ABI
// ------------------------------------------------------------------------------------------
extern "C" {

int gaccum_version(void) { return GACCUM_VERSION; }
const char* gaccum_last_error(void) { return g_err.c_str(); }

int gaccum_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}

// optimization.py:29-54, fp32 op order (volatile: one rounding per TF op, no double promotion)
float gaccum_learning_rate(double init_lr, int64_t num_train_steps, int64_t num_warmup_steps,
                           int64_t global_step) {
  volatile float lr0 = (float)init_lr;
  volatile float gs = (float)global_step;
  volatile float ds = (float)num_train_steps;
  if (gs > ds) gs = ds;
  volatile float p = gs / ds;
  volatile float omp = 1.0f - p;
  volatile float lr = lr0 * omp;
  if (num_warmup_steps) {
    const int32_t gi = (int32_t)global_step, wi = (int32_t)num_warmup_steps;
    volatile float pct = (float)gi / (float)wi;
    volatile float wlr = (float)init_lr * pct;
    volatile float isw = gi < wi ? 1.0f : 0.0f;
    volatile float x = (1.0f - isw) * lr;
    volatile float y = isw * wlr;
    lr = x + y;
  }
  return lr;
}

int gaccum_is_apply_step(int64_t global_step, int32_t accum_n) {
  if (accum_n <= 0) return 0;
  return ((int32_t)global_step % accum_n) == 0;   // optimization.py:77,91
}

int gaccum_decay_mask(int32_t T, const char* const* names, double weight_decay_rate,
                      const char* const* exclude, int32_t num_exclude, uint8_t* out) {
  if (T < 0 || (T > 0 && (!names || !out))) return fail(GACCUM_EINVAL, "bad arguments to gaccum_decay_mask");
  std::vector<regex_t> res((size_t)std::max(0, num_exclude));
  int compiled = 0;
  int rc = GACCUM_OK;
  for (; compiled < num_exclude; ++compiled) {
    if (!exclude || !exclude[compiled] || regcomp(&res[compiled], exclude[compiled], REG_EXTENDED | REG_NOSUB) != 0) {
      rc = fail(GACCUM_EINVAL, "exclude[%d] is not a valid regular expression", compiled);
      break;
    }
  }
  if (rc == GACCUM_OK) {
    for (int32_t t = 0; t < T; ++t) {
      std::string nm = names[t] ? names[t] : "";
      // optimization.py:189-194 -- strip ":<digits>"
      size_t c = nm.rfind(':');
      if (c != std::string::npos && c + 1 < nm.size() &&
          std::all_of(nm.begin() + c + 1, nm.end(), [](char ch) { return ch >= '0' && ch <= '9'; }))
        nm.resize(c);
      uint8_t use = weight_decay_rate != 0.0;      // optimization.py:181 `if not self.weight_decay_rate`
      for (int i = 0; use && i < num_exclude; ++i)
        if (regexec(&res[i], nm.c_str(), 0, nullptr, 0) == 0) use = 0;   // :183-186 re.search
      out[t] = use;
    }
  }
  for (int i = 0; i < compiled; ++i) regfree(&res[i]);
  return rc;
}

int gaccum_plan_create(gaccum_plan** out, int32_t T, const int64_t* numels, const uint8_t* decay,
                       const gaccum_hparams* hp, int32_t device) {
  if (!out) return fail(GACCUM_EINVAL, "out is NULL");
  *out = nullptr;
  if (T < 0 || (T > 0 && !numels)) return fail(GACCUM_EINVAL, "bad tensor list");
  if (!hp) return fail(GACCUM_EINVAL, "hp is NULL");
  if (hp->variant != GACCUM_ADAM_WEIGHT_DECAY && hp->variant != GACCUM_ADAM && hp->variant != GACCUM_LAMB)
    return fail(GACCUM_EINVAL, "unknown optimizer variant %d", hp->variant);
  if (hp->reserved != 0) return fail(GACCUM_EINVAL, "reserved fields must be 0");
  if (T > kCapLarge)
    return fail(GACCUM_EINVAL, "%d tensors exceed the %d-entry pointer table; use the packed entry point with one slab", T, kCapLarge);
  gaccum_plan* pl = new (std::nothrow) gaccum_plan();
  if (!pl) return fail(GACCUM_ENOMEM, "out of host memory");
  pl->T = T;
  pl->hp = *hp;
  pl->numel.assign(numels, numels + T);
  pl->decay.assign((size_t)T, 0);
  if (hp->variant != GACCUM_ADAM && decay) pl->decay.assign(decay, decay + T);
  if (hp->variant == GACCUM_LAMB) pl->adapt.assign((size_t)T, 1);   // every tensor adapts unless told otherwise
  pl->lr_mult.assign((size_t)T, 1.0f);
  if (int rc = build_layout(pl)) { delete pl; return rc; }
  pl->device = -1;
  if (device >= 0) {
    int n = gaccum_device_count();
    if (device >= n) { delete pl; return fail(GACCUM_ENODEVICE, "CUDA device %d requested but %d device(s) visible; libgaccum has no CPU fallback", device, n); }
    DeviceGuard guard(device);
    cudaDeviceProp prop{};
    cudaError_t e = cudaGetDeviceProperties(&prop, device);
    if (e == cudaSuccess && !prop.cooperativeLaunch) e = cudaErrorNotSupported;
    const size_t tb = std::max<size_t>(1, pl->tiles.size()) * sizeof(TileDesc);
    pl->num_sms = prop.multiProcessorCount;
    pl->max_grid = pl->num_sms * 16;
    if (e == cudaSuccess) e = cudaMalloc(&pl->d_tiles, tb);
    if (e == cudaSuccess && !pl->tiles.empty())
      e = cudaMemcpy(pl->d_tiles, pl->tiles.data(), pl->tiles.size() * sizeof(TileDesc), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMalloc(&pl->d_partials, sizeof(double) * (size_t)pl->max_grid);
    if (e == cudaSuccess) e = cudaMalloc(&pl->d_dp_sync, sizeof(uint32_t) * 8);
    if (e == cudaSuccess) e = cudaMemset(pl->d_dp_sync, 0, sizeof(uint32_t) * 8);
    if (e == cudaSuccess) e = cudaMalloc(&pl->d_barrier, sizeof(unsigned long long));
    if (e == cudaSuccess) e = cudaMemset(pl->d_barrier, 0, sizeof(unsigned long long));
    if (e == cudaSuccess) e = cudaMalloc(&pl->d_counters, 2 * sizeof(LaunchCounters));
    if (e == cudaSuccess) e = cudaMemset(pl->d_counters, 0, 2 * sizeof(LaunchCounters));
#ifdef GACCUM_EXPERIMENTS
    if (e == cudaSuccess) e = cudaMalloc(&pl->d_debug, sizeof(unsigned long long) * 16 * (size_t)pl->max_grid);
    if (e == cudaSuccess) e = cudaMemset(pl->d_debug, 0, sizeof(unsigned long long) * 16 * (size_t)pl->max_grid);
#endif
    if (e == cudaSuccess) e = cudaMalloc(&pl->d_stats, sizeof(gaccum_stats));
    if (e == cudaSuccess) e = cudaMemset(pl->d_stats, 0, sizeof(gaccum_stats));
    if (e == cudaSuccess) e = cudaMalloc(&pl->d_done, sizeof(unsigned int));
    if (e == cudaSuccess) e = cudaMemset(pl->d_done, 0, sizeof(unsigned int));
    if (e == cudaSuccess) e = cudaMalloc(&pl->d_reset, 8 * sizeof(unsigned int));
    if (e == cudaSuccess) e = cudaMemset(pl->d_reset, 0, 8 * sizeof(unsigned int));
    if (e == cudaSuccess) e = cudaMalloc(&pl->d_lr_mult, (size_t)std::max(1, T) * sizeof(float));
    if (e == cudaSuccess && T > 0)
      e = cudaMemcpy(pl->d_lr_mult, pl->lr_mult.data(), (size_t)T * sizeof(float), cudaMemcpyHostToDevice);
    if (hp->variant == GACCUM_LAMB) {
      const size_t nt = (size_t)std::max(1, T);
      const std::vector<float> ones(nt, 1.0f);
      if (e == cudaSuccess) e = cudaMalloc(&pl->d_adapt, nt);
      if (e == cudaSuccess && T > 0) e = cudaMemcpy(pl->d_adapt, pl->adapt.data(), (size_t)T, cudaMemcpyHostToDevice);
      if (e == cudaSuccess) e = cudaMalloc(&pl->d_lamb_acc, 2 * nt * sizeof(LambTensorAcc));
      if (e == cudaSuccess) e = cudaMemset(pl->d_lamb_acc, 0, 2 * nt * sizeof(LambTensorAcc));
      if (e == cudaSuccess) e = cudaMalloc(&pl->d_ratios, nt * sizeof(float));
      if (e == cudaSuccess) e = cudaMemcpy(pl->d_ratios, ones.data(), nt * sizeof(float), cudaMemcpyHostToDevice);
    }
    if (e != cudaSuccess) {
      free_plan_device(pl);
      delete pl;
      return fail(GACCUM_ECUDA, "plan device setup failed: %s", cudaGetErrorString(e));
    }
    pl->device = device;
  }
  *out = pl;
  return GACCUM_OK;
}

int gaccum_plan_destroy(gaccum_plan* pl) {
  if (!pl) return GACCUM_OK;
  if (pl->device >= 0) {
    DeviceGuard guard(pl->device);
    free_plan_device(pl);
  }
  delete pl;
  return GACCUM_OK;
}

int64_t gaccum_padded_size(const gaccum_plan* pl) { return pl ? pl->padded : fail(GACCUM_EINVAL, "plan is NULL"); }
int32_t gaccum_num_tensors(const gaccum_plan* pl) { return pl ? pl->T : fail(GACCUM_EINVAL, "plan is NULL"); }
int64_t gaccum_num_elements(const gaccum_plan* pl) { return pl ? pl->P : fail(GACCUM_EINVAL, "plan is NULL"); }
int32_t gaccum_num_tiles(const gaccum_plan* pl) { return pl ? (int32_t)pl->tiles.size() : fail(GACCUM_EINVAL, "plan is NULL"); }

int gaccum_offsets(const gaccum_plan* pl, int64_t* out) {
  if (!pl || (!out && pl->T > 0)) return fail(GACCUM_EINVAL, "bad arguments to gaccum_offsets");
  std::copy(pl->offset.begin(), pl->offset.end(), out);
  return GACCUM_OK;
}

int64_t gaccum_algorithmic_bytes(const gaccum_plan* pl, int32_t is_apply) {
  if (!pl) return fail(GACCUM_EINVAL, "plan is NULL");
  // accumulate: read G, read a, write a.  apply: read G,a,p,m,v + write p,m,v,a  (SURVEY.md 8(d))
  // The first accumulate of a window does not read a (8 B x P), so a window of N >= 2 moves (8 + 12(N-2) + 36) B x P.
  // The plan does not know N: the accumulate figure is the 12 B x P of the other accumulate steps.
  // 16-bit model: G is 2 bytes (accumulate 10 B x P); the apply reads G 2 + a, p, m, v 16 and writes p, m, v, a 16 +
  // the 2-byte model copy (36 B x P).
  // GACCUM_LAMB apply: those 36 B, plus p read a second time (phase 3) and u written and read back: 48 B x P (a 16-bit
  // plan the same).  Phase 1's a' round trip is not counted, as the clip-apply's is not.
  // An EMA plan also reads and writes the average on every apply: + 8 B x P.
  const int64_t apply_bytes = (pl->hp.variant == GACCUM_LAMB ? 48 : 36) + (pl->ema_on ? 8 : 0);
  if (pl->master) return pl->P * (is_apply ? apply_bytes : 10);
  return pl->P * (is_apply ? apply_bytes : 12);
}

// true iff x is 2^k for an integer k in [lo, hi]
static bool pow2_in(double x, int lo, int hi) {
  if (!(x > 0.0) || !std::isfinite(x)) return false;
  int e = 0;
  const double f = std::frexp(x, &e);   // x = f * 2^e, f in [0.5, 1)
  return f == 0.5 && e - 1 >= lo && e - 1 <= hi;
}

int gaccum_plan_set_loss_scale(gaccum_plan* pl, const gaccum_loss_scale_config* cfg, gaccum_loss_scale_state* device_state) {
  if (!pl) return fail(GACCUM_EINVAL, "plan is NULL");
  if (!cfg) return fail(GACCUM_EINVAL, "cfg is NULL");
  if (!device_state || !aligned16_host(device_state))
    return fail(GACCUM_EINVAL, "device_state must be a 16-byte aligned device pointer");
  if (pl->computed) return fail(GACCUM_EINVAL, "loss scaling can only be set before the plan's first compute call");
  if (!pow2_in(cfg->initial_scale, 0, 127))
    return fail(GACCUM_EINVAL, "initial_scale must be a power of two in [1, 2^127] (got %g)", cfg->initial_scale);
  if (!pow2_in(cfg->multiplier, 1, 127))
    return fail(GACCUM_EINVAL, "multiplier must be a power of two in [2, 2^127] (got %g)", cfg->multiplier);
  if (cfg->growth_interval < 1) return fail(GACCUM_EINVAL, "growth_interval must be >= 1 (got %d)", cfg->growth_interval);
  if (cfg->reserved != 0) return fail(GACCUM_EINVAL, "reserved fields must be 0");
  static_assert(sizeof(gaccum_loss_scale_state) == sizeof(LossScaleState), "header and kernel disagree");
  pl->ls_cfg = *cfg;
  pl->ls_state = device_state;
  pl->ls_on = true;
  return GACCUM_OK;
}

int gaccum_plan_set_param_dtype(gaccum_plan* pl, int32_t dtype, float* master_slab) {
  if (!pl) return fail(GACCUM_EINVAL, "plan is NULL");
  if (dtype != GACCUM_DTYPE_BF16 && dtype != GACCUM_DTYPE_F16)
    return fail(GACCUM_EINVAL, "dtype must be GACCUM_DTYPE_BF16 or GACCUM_DTYPE_F16 (got %d)", dtype);
  if (!master_slab || !aligned16_host(master_slab))
    return fail(GACCUM_EINVAL, "master_slab must be a 16-byte aligned device pointer");
  if (pl->computed) return fail(GACCUM_EINVAL, "the parameter dtype can only be set before the plan's first compute call");
  pl->param_dtype = dtype;
  pl->master = master_slab;
  return GACCUM_OK;
}

int gaccum_plan_set_layer_adaptation(gaccum_plan* pl, const uint8_t* adapt) {
  if (!pl) return fail(GACCUM_EINVAL, "plan is NULL");
  if (pl->hp.variant != GACCUM_LAMB) return fail(GACCUM_EINVAL, "layer adaptation is a GACCUM_LAMB setting (plan variant %d)", pl->hp.variant);
  if (!adapt && pl->T > 0) return fail(GACCUM_EINVAL, "adapt is NULL");
  if (pl->computed) return fail(GACCUM_EINVAL, "layer adaptation can only be set before the plan's first compute call");
  for (int32_t t = 0; t < pl->T; ++t) pl->adapt[t] = adapt[t] ? 1 : 0;
  if (pl->device >= 0 && pl->T > 0) {
    DeviceGuard guard(pl->device);
    CUDA_TRY(cudaMemcpy(pl->d_adapt, pl->adapt.data(), (size_t)pl->T, cudaMemcpyHostToDevice));
  }
  return GACCUM_OK;
}

int gaccum_read_trust_ratios(gaccum_plan* pl, float* host_out, gaccum_stream_t stream) {
  if (!pl || !host_out) return fail(GACCUM_EINVAL, "bad arguments to gaccum_read_trust_ratios");
  if (pl->hp.variant != GACCUM_LAMB) return fail(GACCUM_EINVAL, "trust ratios exist on GACCUM_LAMB plans only (plan variant %d)", pl->hp.variant);
  if (pl->device < 0) return fail(GACCUM_ENODEVICE, "layout-only plan has no trust ratios");
  if (pl->T == 0) return GACCUM_OK;
  DeviceGuard guard(pl->device);
  CUDA_TRY(cudaMemcpyAsync(host_out, pl->d_ratios, sizeof(float) * (size_t)pl->T, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  return GACCUM_OK;
}

int gaccum_plan_set_ema(gaccum_plan* pl, const gaccum_ema_config* cfg, float* ema_slab, gaccum_ema_state* device_state) {
  if (!pl) return fail(GACCUM_EINVAL, "plan is NULL");
  if (!cfg) return fail(GACCUM_EINVAL, "cfg is NULL");
  if (!ema_slab || !aligned16_host(ema_slab)) return fail(GACCUM_EINVAL, "ema_slab must be a 16-byte aligned device pointer");
  if (!device_state || !aligned16_host(device_state))
    return fail(GACCUM_EINVAL, "device_state must be a 16-byte aligned device pointer");
  if (pl->computed) return fail(GACCUM_EINVAL, "the moving average can only be set before the plan's first compute call");
  if (!(cfg->decay >= 0.0 && cfg->decay <= 1.0)) return fail(GACCUM_EINVAL, "decay must be in [0, 1] (got %g)", cfg->decay);
  if (cfg->num_updates != 0 && cfg->num_updates != 1) return fail(GACCUM_EINVAL, "num_updates must be 0 or 1 (got %d)", cfg->num_updates);
  if (cfg->reserved != 0) return fail(GACCUM_EINVAL, "reserved fields must be 0");
  static_assert(sizeof(gaccum_ema_state) == sizeof(EmaState), "header and kernel disagree");
  pl->ema_cfg = *cfg;
  pl->ema_slab = ema_slab;
  pl->ema_state = device_state;
  pl->ema_on = true;
  return GACCUM_OK;
}

int gaccum_ema_init(gaccum_plan* pl, gaccum_ema_state* device_state, int64_t num_updates, gaccum_stream_t stream) {
  if (!pl) return fail(GACCUM_EINVAL, "plan is NULL");
  if (!pl->ema_on) return fail(GACCUM_EINVAL, "this plan keeps no moving average (gaccum_plan_set_ema)");
  if (device_state != pl->ema_state)
    return fail(GACCUM_EINVAL, "device_state is not the state block given to gaccum_plan_set_ema, which the apply reads");
  if (num_updates < 0) return fail(GACCUM_EINVAL, "num_updates must be >= 0 (got %lld)", (long long)num_updates);
  if (pl->device < 0) return fail(GACCUM_ENODEVICE, "layout-only plan (device=-1): a CUDA device is required");
  DeviceGuard guard(pl->device);
  ema_init_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(reinterpret_cast<EmaState*>(device_state), (long long)num_updates);
  CUDA_TRY(cudaGetLastError());
  return GACCUM_OK;
}

int gaccum_plan_set_lr_multipliers(gaccum_plan* pl, const float* mult) {
  if (!pl) return fail(GACCUM_EINVAL, "plan is NULL");
  if (!mult && pl->T > 0) return fail(GACCUM_EINVAL, "mult is NULL");
  if (pl->computed) return fail(GACCUM_EINVAL, "learning-rate multipliers can only be set before the plan's first compute call");
  for (int32_t t = 0; t < pl->T; ++t)
    if (!(std::isfinite(mult[t]) && mult[t] >= 0.0f))
      return fail(GACCUM_EINVAL, "mult[%d] = %g: learning-rate multipliers must be finite and >= 0", t, (double)mult[t]);
  if (pl->device >= 0 && pl->T > 0) {
    DeviceGuard guard(pl->device);
    CUDA_TRY(cudaMemcpy(pl->d_lr_mult, mult, sizeof(float) * (size_t)pl->T, cudaMemcpyHostToDevice));
  }
  pl->lr_mult.assign(mult, mult + pl->T);
  pl->lr_mult_set = true;
  return GACCUM_OK;
}

int gaccum_plan_set_window_weight(gaccum_plan* pl, gaccum_window_weight_state* state) {
  if (!pl) return fail(GACCUM_EINVAL, "plan is NULL");
  if (!state || !aligned16_host(state)) return fail(GACCUM_EINVAL, "state must be a 16-byte aligned device pointer");
  if (pl->computed) return fail(GACCUM_EINVAL, "the window weight can only be set before the plan's first compute call");
  static_assert(sizeof(gaccum_window_weight_state) == sizeof(WindowWeightState), "header and kernel disagree");
  pl->ww_state = state;
  return GACCUM_OK;
}

int gaccum_loss_scale_init(gaccum_plan* pl, gaccum_loss_scale_state* device_state, gaccum_stream_t stream) {
  if (!pl) return fail(GACCUM_EINVAL, "plan is NULL");
  if (!pl->ls_on) return fail(GACCUM_EINVAL, "loss scaling is not set on this plan (gaccum_plan_set_loss_scale)");
  if (!device_state || !aligned16_host(device_state))
    return fail(GACCUM_EINVAL, "device_state must be a 16-byte aligned device pointer");
  if (pl->device < 0) return fail(GACCUM_ENODEVICE, "layout-only plan (device=-1): a CUDA device is required");
  DeviceGuard guard(pl->device);
  loss_scale_init_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(reinterpret_cast<LossScaleState*>(device_state),
                                                           (float)pl->ls_cfg.initial_scale, (float)pl->hp.beta1,
                                                           (float)pl->hp.beta2);
  CUDA_TRY(cudaGetLastError());
  return GACCUM_OK;
}

int gaccum_plan_set_device_schedule(gaccum_plan* pl, const gaccum_schedule_config* cfg, gaccum_schedule_state* block) {
  if (!pl) return fail(GACCUM_EINVAL, "plan is NULL");
  if (!cfg) return fail(GACCUM_EINVAL, "cfg is NULL");
  if (!block || !aligned16_host(block)) return fail(GACCUM_EINVAL, "block must be a 16-byte aligned device pointer");
  if (pl->computed) return fail(GACCUM_EINVAL, "the device schedule can only be set before the plan's first compute call");
  if (!std::isfinite(cfg->init_lr)) return fail(GACCUM_EINVAL, "init_lr must be finite (got %g)", cfg->init_lr);
  if (cfg->num_train_steps < 0 || cfg->num_warmup_steps < 0)
    return fail(GACCUM_EINVAL, "num_train_steps and num_warmup_steps must be >= 0 (got %lld, %lld)",
                (long long)cfg->num_train_steps, (long long)cfg->num_warmup_steps);
  if (cfg->end_lr != 0.0 || cfg->power != 1.0)
    return fail(GACCUM_EINVAL, "the device schedule is create_optimizer's: end_lr must be 0 and power 1 (got %g, %g)",
                cfg->end_lr, cfg->power);
  static_assert(sizeof(gaccum_schedule_state) == sizeof(ScheduleState), "header and kernel disagree");
  pl->sched_cfg = *cfg;
  pl->sched_state = block;
  return GACCUM_OK;
}

int gaccum_schedule_init(gaccum_plan* pl, gaccum_schedule_state* block, int64_t global_step, float beta1_power,
                         float beta2_power, gaccum_stream_t stream) {
  if (!pl) return fail(GACCUM_EINVAL, "plan is NULL");
  if (!pl->sched_state) return fail(GACCUM_EINVAL, "this plan has no device schedule (gaccum_plan_set_device_schedule)");
  if (block != pl->sched_state)
    return fail(GACCUM_EINVAL, "block is not the one given to gaccum_plan_set_device_schedule, which the launches read");
  if (global_step < 0) return fail(GACCUM_EINVAL, "global_step must be >= 0 (got %lld)", (long long)global_step);
  if (pl->device < 0) return fail(GACCUM_ENODEVICE, "layout-only plan (device=-1): a CUDA device is required");
  ScheduleState s{};
  s.global_step = (long long)global_step;
  s.num_train_steps = (long long)pl->sched_cfg.num_train_steps;
  s.num_warmup_steps = (long long)pl->sched_cfg.num_warmup_steps;
  s.init_lr = (float)pl->sched_cfg.init_lr;
  s.end_lr = (float)pl->sched_cfg.end_lr;
  s.power = (float)pl->sched_cfg.power;
  if (!pl->ls_on) {          // under loss scaling the beta powers live in the loss-scaling block
    s.beta1_power = beta1_power;
    s.beta2_power = beta2_power;
  }
  DeviceGuard guard(pl->device);
  // a copy from pageable memory: stream-ordered, and `s` is staged before the call returns
  CUDA_TRY(cudaMemcpyAsync(block, &s, sizeof s, cudaMemcpyHostToDevice, (cudaStream_t)stream));
  return GACCUM_OK;
}

int gaccum_plan_set_lr_table(gaccum_plan* pl, const float* device_table, int64_t length) {
  if (!pl) return fail(GACCUM_EINVAL, "plan is NULL");
  if (!device_table) return fail(GACCUM_EINVAL, "device_table is NULL");
  if (length < 1) return fail(GACCUM_EINVAL, "length must be >= 1 (got %lld)", (long long)length);
  if (((uintptr_t)device_table & 3u) != 0) return fail(GACCUM_EINVAL, "device_table must be a 4-byte aligned device pointer");
  if (pl->device < 0) return fail(GACCUM_EINVAL, "layout-only plan (device=-1): a learning-rate table needs a device plan");
  if (pl->computed) return fail(GACCUM_EINVAL, "the learning-rate table can only be set before the plan's first compute call");
  pl->lr_table.table = device_table;
  pl->lr_table.length = length;
  return GACCUM_OK;
}

int gaccum_plan_set_tensor_norms(gaccum_plan* pl, float* device_out) {
  if (!pl) return fail(GACCUM_EINVAL, "plan is NULL");
  if (!device_out || !aligned16_host(device_out)) return fail(GACCUM_EINVAL, "device_out must be a 16-byte aligned device pointer");
  if (pl->device < 0) return fail(GACCUM_EINVAL, "layout-only plan (device=-1): per-tensor norms need a device plan");
  if (pl->computed) return fail(GACCUM_EINVAL, "per-tensor norms can only be set before the plan's first compute call");
  // the tables of NormParams: tensor t's tiles and chunks of up to kNormChunk of them
  const int32_t T = pl->T;
  const int64_t nt = (int64_t)pl->tiles.size();
  std::vector<int32_t> tile_begin((size_t)T + 1, 0), chunk_begin((size_t)T + 1, 0), chunk_tensor;
  for (int32_t t = 0; t < T; ++t) {
    const int64_t tiles = (pl->numel[t] + kTile - 1) / kTile;
    tile_begin[t + 1] = tile_begin[t] + (int32_t)tiles;
    const int64_t chunks = (tiles + kNormChunk - 1) / kNormChunk;
    chunk_begin[t + 1] = chunk_begin[t] + (int32_t)chunks;
    chunk_tensor.insert(chunk_tensor.end(), (size_t)chunks, t);
  }
  if (tile_begin[T] != nt) return fail(GACCUM_EINVAL, "internal error: the tile table does not match the tensors");
  const int64_t nc = chunk_begin[T];
  // doubles first (8-byte aligned), then the int32 tables and the counters
  const size_t b_tile = sizeof(double) * (size_t)nt * kNormCols * kNormWarps;
  const size_t b_chunk = sizeof(double) * (size_t)nc * kNormCols;
  const size_t b_ints = sizeof(int32_t) * (2 * ((size_t)T + 1) + 2 * (size_t)nc + (size_t)T);
  DeviceGuard guard(pl->device);
  if (pl->d_norms) { cudaFree(pl->d_norms); pl->d_norms = nullptr; pl->norms = NormParams{}; }
  void* blk = nullptr;
  CUDA_TRY(cudaMalloc(&blk, b_tile + b_chunk + b_ints + 16));
  NormParams np{};
  np.tile_part = reinterpret_cast<double*>(blk);
  np.chunk_part = reinterpret_cast<double*>(reinterpret_cast<char*>(blk) + b_tile);
  int32_t* ints = reinterpret_cast<int32_t*>(reinterpret_cast<char*>(blk) + b_tile + b_chunk);
  np.tile_begin = ints;
  np.chunk_begin = ints + (T + 1);
  np.chunk_tensor = ints + 2 * (T + 1);
  np.chunk_done = reinterpret_cast<unsigned int*>(ints + 2 * (T + 1) + nc);
  np.tensor_done = reinterpret_cast<unsigned int*>(ints + 2 * (T + 1) + 2 * nc);
  np.num_chunks = (int32_t)nc;
  np.out = device_out;
  cudaError_t e = cudaMemset(ints, 0, b_ints);
  if (e == cudaSuccess) e = cudaMemcpy(ints, tile_begin.data(), sizeof(int32_t) * ((size_t)T + 1), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(ints + (T + 1), chunk_begin.data(), sizeof(int32_t) * ((size_t)T + 1), cudaMemcpyHostToDevice);
  if (e == cudaSuccess && nc > 0)
    e = cudaMemcpy(ints + 2 * (T + 1), chunk_tensor.data(), sizeof(int32_t) * (size_t)nc, cudaMemcpyHostToDevice);
  if (e == cudaSuccess && T > 0) e = cudaMemset(device_out, 0, sizeof(float) * kNormCols * (size_t)T);   // 0 before the first apply
  if (e == cudaSuccess) e = cudaStreamSynchronize(0);   // the memsets are stream-ordered: done before the setter returns
  if (e != cudaSuccess) {
    cudaFree(blk);
    return fail(GACCUM_ECUDA, "tensor-norm setup failed: %s", cudaGetErrorString(e));
  }
  pl->d_norms = blk;
  pl->norms = np;
  return GACCUM_OK;
}

static int accumulate_impl(gaccum_plan* pl, const float* const* grads, float* accum,
                           const gaccum_step_args* a, gaccum_stream_t stream) {
  if (int rc = check_compute(pl, accum, nullptr, nullptr, false)) return rc;
  if (!grads) return fail(GACCUM_EINVAL, "grads is NULL");
  DeviceGuard guard(pl->device);
  cudaStream_t st = (cudaStream_t)stream;
  return pl->T <= kCapSmall ? do_accumulate_tab<kCapSmall>(pl, grads, accum, a, st)
                            : do_accumulate_tab<kCapLarge>(pl, grads, accum, a, st);
}

int gaccum_accumulate(gaccum_plan* pl, const float* const* grads, float* accum, gaccum_stream_t stream) {
  // without step arguments the launch cannot check global_step against its branch: a device-scheduled plan steps with
  // gaccum_step
  if (int rc = refuse(pl, kPlanSchedule | kPlanLrTable, "gaccum_accumulate")) return rc;
  return accumulate_impl(pl, grads, accum, nullptr, stream);
}

static int apply_impl(gaccum_plan* pl, const float* const* grads, float* const* params, float* accum,
                      float* m, float* v, const gaccum_step_args* a, gaccum_stream_t stream);

int gaccum_apply(gaccum_plan* pl, const float* const* grads, float* const* params, float* accum,
                 float* m, float* v, const gaccum_step_args* a, gaccum_stream_t stream) {
  if (int rc = refuse(pl, kPlanSchedule | kPlanLrTable, "gaccum_apply")) return rc;
  return apply_impl(pl, grads, params, accum, m, v, a, stream);
}

static int apply_impl(gaccum_plan* pl, const float* const* grads, float* const* params, float* accum,
                      float* m, float* v, const gaccum_step_args* a, gaccum_stream_t stream) {
  if (int rc = check_compute(pl, accum, m, v, true)) return rc;
  if (int rc = check_args(a)) return rc;
  if (!params) return fail(GACCUM_EINVAL, "params is NULL");
  DeviceGuard guard(pl->device);
  cudaStream_t st = (cudaStream_t)stream;
  return pl->T <= kCapSmall ? do_apply_tab<kCapSmall>(pl, grads, params, accum, m, v, a, st)
                            : do_apply_tab<kCapLarge>(pl, grads, params, accum, m, v, a, st);
}

int gaccum_step(gaccum_plan* pl, const float* const* grads, float* const* params, float* accum,
                float* m, float* v, const gaccum_step_args* a, gaccum_stream_t stream) {
  if (int rc = check_args(a)) return rc;
  if (!grads) return fail(GACCUM_EINVAL, "grads is NULL");
  if (gaccum_is_apply_step(a->global_step, a->accum_n)) return apply_impl(pl, grads, params, accum, m, v, a, stream);
  return accumulate_impl(pl, grads, accum, a, stream);
}

int gaccum_plan_set_deferred_reset(gaccum_plan* pl, int32_t on) {
  if (!pl) return fail(GACCUM_EINVAL, "plan is NULL");
  if (pl->device < 0) return fail(GACCUM_EINVAL, "a layout-only plan (device=-1) has no accumulators to reset");
  if (on != 0 && on != 1) return fail(GACCUM_EINVAL, "on must be 0 or 1 (got %d)", on);
  pl->deferred = on != 0;
  return GACCUM_OK;
}

// The first-accumulate kernel with no gradients, no schedule and the plan's own stats block: it stores +0 over every
// tensor while the word is 1, then clears it (accumulate_kernel), and touches no other device state
extern "C++" {
template <int CAP>
static int do_materialize(gaccum_plan* pl, float* accum, cudaStream_t st) {
  KernelParams<CAP>* prm = new (std::nothrow) KernelParams<CAP>();
  if (!prm) return fail(GACCUM_ENOMEM, "out of host memory");
  fill_common(pl, *prm, accum, nullptr, nullptr, nullptr);
  prm->sched.state = nullptr;
  prm->stats = reinterpret_cast<float*>(pl->d_reset + 4);
  const int rc = pl->master ? launch_accumulate<CAP, true>(pl, *prm, true, st) : launch_accumulate<CAP, false>(pl, *prm, true, st);
  delete prm;
  return rc;
}
}  // extern "C++"

int gaccum_accum_materialize(gaccum_plan* pl, float* accum, gaccum_stream_t stream) {
  if (!pl) return fail(GACCUM_EINVAL, "plan is NULL");
  if (pl->device < 0)
    return fail(GACCUM_ENODEVICE, "layout-only plan (device=-1): libgaccum has no CPU fallback, a CUDA device is required");
  if (!accum || !aligned16_host(accum)) return fail(GACCUM_EINVAL, "accum must be a 16-byte aligned device pointer");
  if (!pl->deferred) return GACCUM_OK;      // every apply of this plan stores the zeros itself
  DeviceGuard guard(pl->device);
  cudaStream_t st = (cudaStream_t)stream;
  return pl->T <= kCapSmall ? do_materialize<kCapSmall>(pl, accum, st) : do_materialize<kCapLarge>(pl, accum, st);
}

int gaccum_step_packed(gaccum_plan* pl, const float* grad_slab, float* param_slab, float* accum,
                       float* m, float* v, const gaccum_step_args* a, int32_t force_branch,
                       gaccum_stream_t stream) {
  if (int rc = refuse(pl, kPlanHalf, "gaccum_step_packed")) return rc;
  if (int rc = check_args(a)) return rc;
  if (pl && pl->sched_state && force_branch >= 0)
    return fail(GACCUM_EINVAL, "a device-scheduled plan takes its branch from global_step: force_branch must be -1 (got %d)", force_branch);
  const bool apply = force_branch < 0 ? gaccum_is_apply_step(a->global_step, a->accum_n) != 0 : force_branch != 0;
  if (int rc = check_compute(pl, accum, m, v, apply)) return rc;
  if (grad_slab && !aligned16_host(grad_slab)) return fail(GACCUM_EINVAL, "grad_slab must be 16-byte aligned");
  DeviceGuard guard(pl->device);
  cudaStream_t st = (cudaStream_t)stream;
  KernelParams<0> prm{};
  fill_common(pl, prm, accum, m, v, a);
  prm.dr.accum_zero = nullptr;   // a packed slab (autograd adds into it) always holds real zeros: no deferred reset
  prm.tab.g = grad_slab;
  prm.tab.p = param_slab;
  if (!apply) {
    if (!grad_slab && pl->sched_state) {
      // the gradients are already in accum (PackedTrainOp): one CTA only advances the device schedule
      prm.num_tiles = 0;
      return launch_accumulate(pl, prm, false, st);
    }
    if (!grad_slab) return fail(GACCUM_EINVAL, "grad_slab is NULL on an accumulate step");
    // a forced branch says nothing about what the previous micro-step did: only the scheduled one may skip reading a
    return launch_accumulate(pl, prm, force_branch < 0 && first_of_window(a), st);
  }
  if (!param_slab || !aligned16_host(param_slab)) return fail(GACCUM_EINVAL, "param_slab must be a 16-byte aligned device pointer");
  return pl->ema_on ? launch_apply<0, false, true>(pl, prm, st) : launch_apply<0, false, false>(pl, prm, st);
}

// contiguous tile ranges with (nearly) equal element counts: boundary r = first tile whose cumulative
// element count reaches r * P / world
static void shard_bounds(const gaccum_plan* pl, int world, int* bounds /* world + 1 */) {
  const int nt = (int)pl->tiles.size();
  int64_t cum = 0;
  int r = 1;
  bounds[0] = 0;
  for (int t = 0; t < nt && r < world; ++t) {
    cum += pl->tiles[t].len;
    while (r < world && cum >= (pl->P * r + world - 1) / world) bounds[r++] = t + 1;
  }
  while (r <= world) bounds[r++] = nt;
}
// slab offset (in units of 32 elements) at which tile t starts; t == num_tiles -> end of the slab, which is 2^32 for a
// slab of exactly 2^37 elements: int64, not TileDesc's uint32
static int64_t tile_soff32(const gaccum_plan* pl, int t) {
  return t < (int)pl->tiles.size() ? (int64_t)pl->tiles[t].soff32 : pl->padded / kSlabAlign;
}
// elements of one source region of a staging area = the widest shard's slab span
static int64_t stage_span(const gaccum_plan* pl, int world) {
  int bounds[GACCUM_MAX_RANKS + 1];
  shard_bounds(pl, world, bounds);
  int64_t span = 0;
  for (int r = 0; r < world; ++r)
    span = std::max<int64_t>(span, ((int64_t)tile_soff32(pl, bounds[r + 1]) - (int64_t)tile_soff32(pl, bounds[r])) * kSlabAlign);
  return std::max<int64_t>(span, kSlabAlign);
}

int gaccum_dp_shard_range(const gaccum_plan* pl, int32_t world, int32_t rank, int32_t* tile_lo,
                          int32_t* tile_hi, int64_t* num_elements) {
  if (!pl || !tile_lo || !tile_hi) return fail(GACCUM_EINVAL, "bad arguments to gaccum_dp_shard_range");
  if (world < 1 || world > GACCUM_MAX_RANKS || rank < 0 || rank >= world)
    return fail(GACCUM_EINVAL, "world must be 1..%d and 0 <= rank < world (got world=%d rank=%d)", GACCUM_MAX_RANKS, world, rank);
  int bounds[GACCUM_MAX_RANKS + 1];
  shard_bounds(pl, world, bounds);
  *tile_lo = bounds[rank];
  *tile_hi = bounds[rank + 1];
  if (num_elements) {
    int64_t e = 0;
    for (int t = bounds[rank]; t < bounds[rank + 1]; ++t) e += pl->tiles[t].len;
    *num_elements = e;
  }
  return GACCUM_OK;
}

int64_t gaccum_dp_stage_elements(const gaccum_plan* pl, int32_t world) {
  if (!pl) return fail(GACCUM_EINVAL, "plan is NULL");
  if (world < 2 || world > GACCUM_MAX_RANKS) return fail(GACCUM_EINVAL, "world must be 2..%d", GACCUM_MAX_RANKS);
  return stage_span(pl, world) * (world - 1);
}

extern "C++" {
template <int CAP>
static int do_apply_dp(gaccum_plan* pl, const gaccum_dp_comm* comm, const float* const* grads, float* m, float* v,
                       const gaccum_step_args* a, uint32_t epoch, cudaStream_t st) {
  DpParams<CAP>* prm = new (std::nothrow) DpParams<CAP>();
  if (!prm) return fail(GACCUM_ENOMEM, "out of host memory");
  const int W = comm->world;
  for (int w = 0; w < W; ++w) {
    prm->param[w] = comm->param_peers[w];
    prm->stage[w] = comm->stage_peers[w];
    prm->ctrl[w] = comm->ctrl_peers[w];
  }
  prm->tiles = pl->d_tiles;
  prm->num_tiles = (int32_t)pl->tiles.size();
  int bounds[GACCUM_MAX_RANKS + 1];
  shard_bounds(pl, W, bounds);
  // the kernel reads the base of a rank that owns tiles only: a tile start, which fits 32 bits
  for (int r = 0; r <= W; ++r) { prm->bounds[r] = bounds[r]; prm->shard_base32[r] = (uint32_t)tile_soff32(pl, bounds[r]); }
  prm->stage_span = stage_span(pl, W);
  prm->accum = comm->accum;
  prm->m = m;
  prm->v = v;
  prm->partials = pl->d_partials;
  prm->stats = pl->d_stats;
  prm->sync = pl->d_dp_sync;
#ifdef GACCUM_EXPERIMENTS
  prm->debug = pl->d_debug;
#endif
  prm->sc = make_scalars(pl->hp, a);
  prm->rank = comm->rank;
  prm->world = W;
  prm->epoch = epoch;
  for (int32_t t = 0; t < pl->T; ++t) prm->tab.g[t] = grads ? grads[t] : nullptr;
  const void* fn = pl->hp.variant == GACCUM_ADAM ? (const void*)&dp_apply_kernel<1, CAP> : (const void*)&dp_apply_kernel<0, CAP>;
  int per_sm = 0;
  int rc = fit(pl, fn, "dp_apply_kernel", kThreads, 0, 1, &per_sm);
  if (rc == GACCUM_OK) {
    const int grid = std::max(1, std::min({per_sm * pl->num_sms, pl->max_grid, prm->num_tiles}));
    void* args[] = {(void*)prm};
    cudaError_t e = cudaLaunchCooperativeKernel(fn, dim3(grid), dim3(kThreads), args, 0, st);
    if (e != cudaSuccess) rc = fail(GACCUM_ECUDA, "cudaLaunchCooperativeKernel(dp_apply_kernel) failed: %s", cudaGetErrorString(e));
  }
  delete prm;
  return rc;
}
}  // extern "C++"

int gaccum_apply_dp(gaccum_plan* pl, const gaccum_dp_comm* comm, const float* const* grads, float* m, float* v,
                    const gaccum_step_args* a, uint32_t epoch, gaccum_stream_t stream) {
  if (int rc = refuse(pl, kPlanAll, "the fused data-parallel apply")) return rc;
  if (!comm) return fail(GACCUM_EINVAL, "comm is NULL");
  if (comm->world < 2 || comm->world > GACCUM_MAX_RANKS || comm->rank < 0 || comm->rank >= comm->world)
    return fail(GACCUM_EINVAL, "world must be 2..%d and 0 <= rank < world", GACCUM_MAX_RANKS);
  if (epoch == 0) return fail(GACCUM_EINVAL, "epoch must be non-zero");
  if (int rc = check_args(a)) return rc;
  if (int rc = check_compute(pl, comm->accum, m, v, true)) return rc;
  static_assert(kMaxRanks == GACCUM_MAX_RANKS && kCtrlBytes == GACCUM_DP_CTRL_BYTES, "header and kernel disagree");
  if (comm->stage_elements < stage_span(pl, comm->world) * (comm->world - 1))
    return fail(GACCUM_EINVAL, "staging areas hold %lld elements, gaccum_dp_stage_elements() asks for %lld",
                (long long)comm->stage_elements, (long long)(stage_span(pl, comm->world) * (comm->world - 1)));
  for (int w = 0; w < comm->world; ++w)
    if (!comm->param_peers[w] || !comm->stage_peers[w] || !comm->ctrl_peers[w] ||
        !aligned16_host(comm->param_peers[w]) || !aligned16_host(comm->stage_peers[w]))
      return fail(GACCUM_EINVAL, "peer pointers of rank %d must be non-NULL and 16-byte aligned", w);
  DeviceGuard guard(pl->device);
  cudaStream_t st = (cudaStream_t)stream;
  return pl->T <= kCapSmall ? do_apply_dp<kCapSmall>(pl, comm, grads, m, v, a, epoch, st)
                            : do_apply_dp<kCapLarge>(pl, comm, grads, m, v, a, epoch, st);
}

int gaccum_step_dp(gaccum_plan* pl, const gaccum_dp_comm* comm, const float* const* grads, float* m, float* v,
                   const gaccum_step_args* a, uint32_t epoch, gaccum_stream_t stream) {
  if (int rc = refuse(pl, kPlanAll, "the fused data-parallel step")) return rc;
  if (!comm) return fail(GACCUM_EINVAL, "comm is NULL");
  if (int rc = check_args(a)) return rc;
  if (!grads) return fail(GACCUM_EINVAL, "grads is NULL");
  if (gaccum_is_apply_step(a->global_step, a->accum_n)) return gaccum_apply_dp(pl, comm, grads, m, v, a, epoch, stream);
  return accumulate_impl(pl, grads, comm->accum, a, stream);      // rank-local: no bytes cross NVLink
}

// ------------------------------------------------------------------------------------------
// host-buffer session
// ------------------------------------------------------------------------------------------
struct gaccum_host_session {
  gaccum_plan* plan = nullptr;
  float *d_params = nullptr, *d_accum = nullptr, *d_m = nullptr, *d_v = nullptr;
  float* d_stage[2] = {nullptr, nullptr};                    // H2D staging of the gradients, double-buffered
  std::vector<const float*> stage_ptrs[2];                   // per-tensor views of the staging slabs (pointer table of the DP kernel)
  cudaStream_t compute = nullptr, h2d = nullptr, d2h = nullptr;
  cudaEvent_t buf_free[2] = {nullptr, nullptr}, h2d_done[2] = {nullptr, nullptr}, k_done = nullptr, d2h_done = nullptr;
  uint64_t calls = 0;
  // data parallel (gaccum_host_session_dp_export / _connect)
  int dp_rank = 0, dp_world = 1;
  float* d_dp_stage = nullptr;                               // this rank's reduce-scatter staging area (peer-written)
  uint32_t* d_dp_ctrl = nullptr;
  int64_t dp_stage_elements = 0;
  gaccum_dp_comm comm{};
  std::vector<void*> ipc_opened;
  uint32_t dp_epoch = 0;
};

// One cudaMemcpyAsync per RUN of tensors whose host addresses are laid out like the device slab (same distance
// between consecutive tensors on both sides, padding included): a caller that keeps its gradients / parameters
// in one pinned arena with the plan's offsets gets a single copy per direction instead of one per tensor
// (every copy costs a copy-engine gap: many small copies hold the link well below what one large copy reaches).
extern "C++" {
template <typename HostPtr, typename F>
static int for_each_run(const gaccum_plan* pl, HostPtr const* host, F&& copy /* (t0, host_ptr, dev_offset, elements) -> cudaError_t */) {
  int32_t t = 0;
  while (t < pl->T) {
    if (pl->numel[t] == 0 || !host[t]) { ++t; continue; }
    const int32_t t0 = t;
    int64_t span = pl->numel[t];
    while (t + 1 < pl->T && host[t + 1] && pl->numel[t + 1] > 0 &&
           (const float*)host[t + 1] - (const float*)host[t0] == pl->offset[t + 1] - pl->offset[t0]) {
      ++t;
      span = pl->offset[t] - pl->offset[t0] + pl->numel[t];
    }
    cudaError_t e = copy(t0, host[t0], pl->offset[t0], span);
    if (e != cudaSuccess) return fail(GACCUM_ECUDA, "host<->device copy failed: %s", cudaGetErrorString(e));
    ++t;
  }
  return GACCUM_OK;
}
}  // extern "C++"

int gaccum_host_session_destroy(gaccum_host_session* s) {
  if (!s) return GACCUM_OK;
  if (s->plan && s->plan->device >= 0) {
    DeviceGuard guard(s->plan->device);
    if (s->compute) cudaStreamSynchronize(s->compute);
    if (s->h2d) cudaStreamSynchronize(s->h2d);
    if (s->d2h) cudaStreamSynchronize(s->d2h);
    for (void* p : s->ipc_opened) cudaIpcCloseMemHandle(p);
    cudaFree(s->d_params); cudaFree(s->d_accum); cudaFree(s->d_m); cudaFree(s->d_v);
    cudaFree(s->d_stage[0]); cudaFree(s->d_stage[1]); cudaFree(s->d_dp_stage); cudaFree(s->d_dp_ctrl);
    for (int i = 0; i < 2; ++i) { if (s->buf_free[i]) cudaEventDestroy(s->buf_free[i]); if (s->h2d_done[i]) cudaEventDestroy(s->h2d_done[i]); }
    if (s->k_done) cudaEventDestroy(s->k_done);
    if (s->d2h_done) cudaEventDestroy(s->d2h_done);
    if (s->compute) cudaStreamDestroy(s->compute);
    if (s->h2d) cudaStreamDestroy(s->h2d);
    if (s->d2h) cudaStreamDestroy(s->d2h);
  }
  delete s;
  return GACCUM_OK;
}

int gaccum_host_session_create(gaccum_host_session** out, gaccum_plan* pl) {
  if (!out) return fail(GACCUM_EINVAL, "out is NULL");
  *out = nullptr;
  if (!pl) return fail(GACCUM_EINVAL, "plan is NULL");
  // host-resident models train in fp32 (no fp16 autocast on the CPU): nothing to loss-scale
  if (int rc = refuse(pl, kPlanAll, "the host-buffer session")) return rc;
  if (pl->device < 0) return fail(GACCUM_ENODEVICE, "layout-only plan (device=-1): libgaccum has no CPU fallback, a CUDA device is required");
  DeviceGuard guard(pl->device);
  gaccum_host_session* s = new (std::nothrow) gaccum_host_session();
  if (!s) return fail(GACCUM_ENOMEM, "out of host memory");
  s->plan = pl;
  const size_t bytes = (size_t)std::max<int64_t>(pl->padded, kSlabAlign) * sizeof(float);
  cudaError_t e = cudaSuccess;
  float** bufs[] = {&s->d_params, &s->d_accum, &s->d_m, &s->d_v, &s->d_stage[0], &s->d_stage[1]};
  for (float** b : bufs) {
    if (e == cudaSuccess) e = cudaMalloc(b, bytes);
    if (e == cudaSuccess) e = cudaMemset(*b, 0, bytes);
  }
  if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&s->compute, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&s->h2d, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&s->d2h, cudaStreamNonBlocking);
  for (int i = 0; i < 2 && e == cudaSuccess; ++i) {
    e = cudaEventCreateWithFlags(&s->buf_free[i], cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&s->h2d_done[i], cudaEventDisableTiming);
  }
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&s->k_done, cudaEventDisableTiming);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&s->d2h_done, cudaEventDisableTiming);
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e != cudaSuccess) {
    gaccum_host_session_destroy(s);
    return fail(GACCUM_ECUDA, "host session setup failed: %s", cudaGetErrorString(e));
  }
  for (int b = 0; b < 2; ++b) {
    s->stage_ptrs[b].resize((size_t)pl->T);
    for (int32_t t = 0; t < pl->T; ++t) s->stage_ptrs[b][t] = s->d_stage[b] + pl->offset[t];
  }
  *out = s;
  return GACCUM_OK;
}

int gaccum_host_session_set_params(gaccum_host_session* s, const float* const* host_params) {
  if (!s || !host_params) return fail(GACCUM_EINVAL, "bad arguments to gaccum_host_session_set_params");
  gaccum_plan* pl = s->plan;
  DeviceGuard guard(pl->device);
  for (int32_t t = 0; t < pl->T; ++t)
    if (pl->numel[t] && !host_params[t]) return fail(GACCUM_EINVAL, "host_params[%d] is NULL", t);
  if (int rc = for_each_run(pl, host_params, [&](int32_t, const float* h, int64_t off, int64_t n) {
        return cudaMemcpyAsync(s->d_params + off, h, (size_t)n * sizeof(float), cudaMemcpyHostToDevice, s->compute);
      })) return rc;
  CUDA_TRY(cudaStreamSynchronize(s->compute));
  return GACCUM_OK;
}

// ---- data parallel over host buffers: every rank's session exports IPC handles of its parameter slab, staging
//      area and control block; the caller exchanges the (plain-byte) records between the ranks with whatever
//      transport it has (MPI, torch.distributed, TF collectives) and hands all of them back ----
int gaccum_host_session_dp_export(gaccum_host_session* s, int32_t world, gaccum_dp_ipc* out) {
  if (!s || !out) return fail(GACCUM_EINVAL, "bad arguments to gaccum_host_session_dp_export");
  if (world < 2 || world > GACCUM_MAX_RANKS) return fail(GACCUM_EINVAL, "world must be 2..%d", GACCUM_MAX_RANKS);
  static_assert(sizeof(cudaIpcMemHandle_t) == GACCUM_IPC_HANDLE_BYTES, "cudaIpcMemHandle_t is 64 bytes");
  gaccum_plan* pl = s->plan;
  DeviceGuard guard(pl->device);
  if (!s->d_dp_stage) {
    s->dp_stage_elements = stage_span(pl, world) * (world - 1);
    CUDA_TRY(cudaMalloc(&s->d_dp_stage, (size_t)s->dp_stage_elements * sizeof(float)));
    CUDA_TRY(cudaMalloc(&s->d_dp_ctrl, GACCUM_DP_CTRL_BYTES));
    CUDA_TRY(cudaMemset(s->d_dp_ctrl, 0, GACCUM_DP_CTRL_BYTES));
    CUDA_TRY(cudaDeviceSynchronize());
  }
  std::memset(out, 0, sizeof *out);
  cudaIpcMemHandle_t h;
  CUDA_TRY(cudaIpcGetMemHandle(&h, s->d_params)); std::memcpy(out->param, &h, sizeof h);
  CUDA_TRY(cudaIpcGetMemHandle(&h, s->d_dp_stage)); std::memcpy(out->stage, &h, sizeof h);
  CUDA_TRY(cudaIpcGetMemHandle(&h, s->d_dp_ctrl)); std::memcpy(out->ctrl, &h, sizeof h);
  out->stage_elements = s->dp_stage_elements;
  out->padded_size = pl->padded;
  return GACCUM_OK;
}

int gaccum_host_session_dp_connect(gaccum_host_session* s, int32_t rank, int32_t world, const gaccum_dp_ipc* all) {
  if (!s || !all) return fail(GACCUM_EINVAL, "bad arguments to gaccum_host_session_dp_connect");
  if (world < 2 || world > GACCUM_MAX_RANKS || rank < 0 || rank >= world) return fail(GACCUM_EINVAL, "world must be 2..%d and 0 <= rank < world", GACCUM_MAX_RANKS);
  if (!s->d_dp_stage) return fail(GACCUM_EINVAL, "call gaccum_host_session_dp_export first");
  gaccum_plan* pl = s->plan;
  DeviceGuard guard(pl->device);
  gaccum_dp_comm c{};
  c.rank = rank; c.world = world; c.accum = s->d_accum; c.stage_elements = s->dp_stage_elements;
  for (int w = 0; w < world; ++w) {
    if (all[w].padded_size != pl->padded || all[w].stage_elements != s->dp_stage_elements)
      return fail(GACCUM_EINVAL, "rank %d exported a different layout (padded %lld vs %lld): all ranks must use the same plan",
                  w, (long long)all[w].padded_size, (long long)pl->padded);
    if (w == rank) { c.param_peers[w] = s->d_params; c.stage_peers[w] = s->d_dp_stage; c.ctrl_peers[w] = s->d_dp_ctrl; continue; }
    void* ptr[3] = {nullptr, nullptr, nullptr};
    const unsigned char* src[3] = {all[w].param, all[w].stage, all[w].ctrl};
    for (int k = 0; k < 3; ++k) {
      cudaIpcMemHandle_t h;
      std::memcpy(&h, src[k], sizeof h);
      cudaError_t e = cudaIpcOpenMemHandle(&ptr[k], h, cudaIpcMemLazyEnablePeerAccess);
      if (e != cudaSuccess) return fail(GACCUM_ECUDA, "cudaIpcOpenMemHandle(rank %d, buffer %d) failed: %s (ranks must be GPUs of one NVLink/PCIe peer domain)", w, k, cudaGetErrorString(e));
      s->ipc_opened.push_back(ptr[k]);
    }
    c.param_peers[w] = (float*)ptr[0]; c.stage_peers[w] = (float*)ptr[1]; c.ctrl_peers[w] = (uint32_t*)ptr[2];
  }
  s->comm = c;
  s->dp_rank = rank; s->dp_world = world;
  return GACCUM_OK;
}

int gaccum_step_host(gaccum_host_session* s, const float* const* host_grads, float* const* host_params_out,
                     const gaccum_step_args* a, gaccum_stats* stats_out) {
  if (!s || !host_grads) return fail(GACCUM_EINVAL, "bad arguments to gaccum_step_host");
  if (int rc = check_args(a)) return rc;
  gaccum_plan* pl = s->plan;
  if (int rc = refuse(pl, kPlanAll, "the host-buffer session")) return rc;
  DeviceGuard guard(pl->device);
  const int b = (int)(s->calls & 1);
  ++s->calls;
  // H2D of this step's gradients into staging buffer b, once the kernel that last read it is done
  CUDA_TRY(cudaStreamWaitEvent(s->h2d, s->buf_free[b], 0));
  if (int rc = for_each_run(pl, host_grads, [&](int32_t, const float* h, int64_t off, int64_t n) {
        return cudaMemcpyAsync(s->d_stage[b] + off, h, (size_t)n * sizeof(float), cudaMemcpyHostToDevice, s->h2d);
      })) return rc;
  for (int32_t t = 0; t < pl->T; ++t)     // tensors without a gradient contribute nothing (optimization.py:132): stage zeros
    if (pl->numel[t] && !host_grads[t])
      CUDA_TRY(cudaMemsetAsync(s->d_stage[b] + pl->offset[t], 0, (size_t)pl->numel[t] * sizeof(float), s->h2d));
  CUDA_TRY(cudaEventRecord(s->h2d_done[b], s->h2d));
  CUDA_TRY(cudaStreamWaitEvent(s->compute, s->h2d_done[b], 0));
  const bool apply = gaccum_is_apply_step(a->global_step, a->accum_n) != 0;
  if (s->dp_world > 1 && apply) {
    // 04:55-62 through host buffers: the fused exchange + apply kernel reads this rank's staged gradients
    if (++s->dp_epoch == 0) s->dp_epoch = 1;
    if (int rc = gaccum_apply_dp(pl, &s->comm, s->stage_ptrs[b].data(), s->d_m, s->d_v, a, s->dp_epoch, s->compute)) return rc;
  } else {
    if (int rc = gaccum_step_packed(pl, s->d_stage[b], s->d_params, s->d_accum, s->d_m, s->d_v, a, -1, s->compute)) return rc;
  }
  CUDA_TRY(cudaEventRecord(s->buf_free[b], s->compute));
  if (stats_out)
    CUDA_TRY(cudaMemcpyAsync(stats_out, pl->d_stats, sizeof(gaccum_stats), cudaMemcpyDeviceToHost, s->compute));
  if (apply && host_params_out) {
    CUDA_TRY(cudaEventRecord(s->k_done, s->compute));
    CUDA_TRY(cudaStreamWaitEvent(s->d2h, s->k_done, 0));
    if (int rc = for_each_run(pl, host_params_out, [&](int32_t, float* h, int64_t off, int64_t n) {
          return cudaMemcpyAsync(h, s->d_params + off, (size_t)n * sizeof(float), cudaMemcpyDeviceToHost, s->d2h);
        })) return rc;
    CUDA_TRY(cudaEventRecord(s->d2h_done, s->d2h));
    CUDA_TRY(cudaStreamWaitEvent(s->compute, s->d2h_done, 0));   // the next apply must not overwrite params mid-copy
  }
  return GACCUM_OK;
}

int gaccum_host_session_sync(gaccum_host_session* s) {
  if (!s) return fail(GACCUM_EINVAL, "session is NULL");
  DeviceGuard guard(s->plan->device);
  CUDA_TRY(cudaStreamSynchronize(s->h2d));
  CUDA_TRY(cudaStreamSynchronize(s->compute));
  CUDA_TRY(cudaStreamSynchronize(s->d2h));
  return GACCUM_OK;
}

int gaccum_host_session_slabs(gaccum_host_session* s, float** out) {
  if (!s || !out) return fail(GACCUM_EINVAL, "bad arguments to gaccum_host_session_slabs");
  out[0] = s->d_params; out[1] = s->d_accum; out[2] = s->d_m; out[3] = s->d_v;
  return GACCUM_OK;
}

#ifdef GACCUM_EXPERIMENTS
// Experiments build only (-DGACCUM_EXPERIMENTS, not declared in gaccum.h): per-CTA timestamps of the last clip-apply launch.
extern "C" __attribute__((visibility("default"))) int gaccum_debug_read(gaccum_plan* pl, unsigned long long* out, int n) {
  if (!pl || !pl->d_debug) return fail(GACCUM_EINVAL, "no debug buffer");
  DeviceGuard guard(pl->device);
  CUDA_TRY(cudaMemcpy(out, pl->d_debug, sizeof(unsigned long long) * (size_t)std::min(n, 16 * pl->max_grid), cudaMemcpyDeviceToHost));
  return GACCUM_OK;
}
#endif

int gaccum_read_stats(gaccum_plan* pl, gaccum_stats* host_out, gaccum_stream_t stream) {
  if (!pl || !host_out) return fail(GACCUM_EINVAL, "bad arguments to gaccum_read_stats");
  if (pl->device < 0) return fail(GACCUM_ENODEVICE, "layout-only plan has no stats");
  DeviceGuard guard(pl->device);
  CUDA_TRY(cudaMemcpyAsync(host_out, pl->d_stats, sizeof(gaccum_stats), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  return GACCUM_OK;
}

}  // extern "C"
