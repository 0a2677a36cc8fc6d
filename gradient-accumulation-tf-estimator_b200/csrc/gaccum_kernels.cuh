// gaccum_kernels.cuh -- sm_90a kernels of the gradient-accumulation train_op.
//
// All kernels walk a static tile table (<= 2048 elements of one tensor per tile), so the work split --
// and therefore every reduction -- is deterministic.
//
//   accumulate_kernel    a += G                                  optimization.py:81,93    (12 B/elem)
//                        one tile per CTA (hardware block scheduler); the first accumulate of a window
//                        stores a = +0 + G without reading a                             (8 B/elem)
//   apply_kernel         the apply branch WITHOUT clipping (plain Adam of the example scripts, or
//                        clip_norm <= 0): a' = a + G; n = a'/N; Adam; a = 0 in a single pass (36 B/elem).
//   apply_clip_kernel    the apply branch WITH tf.clip_by_global_norm                  (36 B/elem)
//                        optimization.py:80-88, 128-177.  The global norm of ALL tensors is needed before
//                        ANY element can be updated: one cooperative launch, two passes around a grid
//                        barrier (described at the kernel).  Its loss-scaled instantiations (kLsClip, kLsNoClip)
//                        also unscale by 1/S and skip the whole window when a' or the norm is not finite; with
//                        clipping off they run the same two passes with the norm and the clip multiply compiled out.
// Arithmetic uses round-to-nearest intrinsics (__fmul_rn, __fadd_rn, __fdiv_rn, __fsqrt_rn) so nvcc
// cannot contract mul+add into FMA: the reference graph is un-fused, one rounding per TF op, and we
// reproduce it bit for bit (the kernels are HBM-bound, the extra flops are free).
//
// 16-bit models (template flag H, scattered pointer tables only): G and the model's weights are bf16 or fp16 (one
// launch-uniform flag, prm.half.bf16), the fp32 master weights are a slab in the plan's layout.  G is widened exactly
// on load, so every fp32 operation is the one the fp32 kernels perform on the upcast gradient; the apply stores the
// master weights and, rounded to nearest-even, the model copy.  accumulate 10 B/elem (first of a window 6), apply 36.
//
// Exponential moving average of the weights (template flag EMA, gaccum_plan_set_ema): every apply kernel also reads the
// average e and stores e - (e - p) * c after p, on applied windows only (+8 B/elem); see EmaParams.
//
// Per-tensor norms (launch-uniform, gaccum_plan_set_tensor_norms): every apply kernel also sums c^2, p^2 and (p - p')^2
// per tile into plan scratch and reduces them per tensor in a fixed order; see NormParams.
#pragma once

#include <cooperative_groups.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace gaccum {
namespace cg = cooperative_groups;

constexpr int kThreads = 256;                    // 8 warps per CTA / per consumer group
constexpr int kUnroll = 2;                       // 128-bit vectors per thread per stream per tile
constexpr int kTile = kThreads * 4 * kUnroll;    // 2048 elements = 8 KB per stream
constexpr int kSlabAlign = 32;                   // tensors start at multiples of 32 elements (128 B)

// One unit of work: <= kTile consecutive elements of ONE tensor (so pointers and the decay flag
// are tile-uniform).  16 bytes, read with a single LDG.128.
struct __align__(16) TileDesc {
  uint32_t tensor_flags;   // bits 0..30 tensor index, bit 31 = apply weight decay (optimization.py:166)
  uint32_t len;            // elements in this tile (1..kTile)
  uint32_t toff;           // element offset inside the tensor (multiple of kTile)
  uint32_t soff32;         // element offset inside the slabs, in units of 32 elements
};

// Scattered inputs arrive as a pointer table that lives in the kernel-parameter (constant)
// space: no device-side table to keep in sync, launches stay re-entrant and graph-capturable.
// CAP = 0 is the packed layout (grads/params are slabs with the same offsets as accum).
template <int CAP>
struct PtrTable {
  const float* g[CAP];
  float* p[CAP];
};
template <>
struct PtrTable<0> {
  const float* g;
  float* p;
};

struct Scalars {
  float nf;      // fp32(N)                                   optimization.py:83
  float inv_nf;  // 1/N when N is a power of two (exact), else 0 -> the kernels divide
  float lr;      // learning rate of this micro-step          optimization.py:29-54
  float b1, b2;  // fp32(beta)                                optimization.py:151,153
  float omb1;    // A: fp32(1.0 - beta1) from double (:152);  B: 1.0f - fp32(beta1)
  float omb2;
  float eps;     //                                           optimization.py:157
  float wd;      //                                           optimization.py:167
  float clip;    //                                           optimization.py:84
  float b1p, b2p;  // GACCUM_ADAM, GACCUM_LAMB: TF1's beta powers of this step (gaccum_step_args; 0 without)
};

// gaccum_loss_scale_state (gaccum.h): caller-owned device memory, written only by the loss-scaled apply launch
struct LossScaleState {
  float scale;                // S, a power of two in [1, 2^127]
  int32_t good_windows;       // applied windows since S last changed
  uint32_t skipped_windows;   // overflowed windows since initialisation
  int32_t last_skipped;       // 1 if the last apply launch skipped its window
  float beta1_power, beta2_power;   // GACCUM_ADAM: TF1's beta powers, advanced on applied windows only
  float reserved[2];
};
static_assert(sizeof(LossScaleState) == 32, "gaccum_loss_scale_state is 32 bytes");

// Loss scaling of one apply launch.  Kept after the pointer table, at the end of KernelParams, so every other member
// sits where it does without loss scaling.
struct LossScaleParams {
  LossScaleState* state;
  float multiplier;           // a power of two >= 2
  int32_t growth_interval;    // applied windows before S grows
};
// The mode of the cooperative apply kernels (MODE): apply_clip_kernel has every mode but kNoClip, lamb_apply_kernel all
constexpr int kNoClip = 0;      // neither clipping nor loss scaling
constexpr int kClip = 1;        // tf.clip_by_global_norm
constexpr int kLsClip = 2;      // loss scaling + tf.clip_by_global_norm
constexpr int kLsNoClip = 3;    // loss scaling without clipping: pass 1 only looks for non-finite elements of a'
__host__ __device__ constexpr bool loss_scaled(int mode) { return mode == kLsClip || mode == kLsNoClip; }

// A 16-bit model (gaccum_plan_set_param_dtype): the pointer table's g[] and p[] point at bf16 or fp16 tensors.  Kept
// after LossScaleParams, so every member of the fp32 instantiations sits where it does without it.
struct HalfParams {
  float* master;      // fp32 master weights, a slab in the plan's layout (16-byte aligned)
  int32_t bf16;       // 1: bf16, 0: fp16
};

// GACCUM_LAMB (gaccum_lamb.cuh): the per-tensor accumulators and the trust ratios
struct LambParams {
  struct LambTensorAcc* acc;   // 2 sets x num_tensors
  float* ratios;           // num_tensors: r of the last applied window (gaccum_read_trust_ratios)
  const uint8_t* adapt;    // num_tensors: 1 = layer adaptation (gaccum_plan_set_layer_adaptation)
  int32_t num_tensors;
};

// gaccum_ema_state (gaccum.h): caller-owned device memory, written by gaccum_ema_init and afterwards only by the apply
// launches of an EMA plan
struct EmaState {
  long long num_updates;   // n: windows averaged so far
  float decay;             // d of the last averaged window
  float reserved;
};
static_assert(sizeof(EmaState) == 16, "gaccum_ema_state is 16 bytes");

// The exponential moving average of the weights (gaccum_plan_set_ema)
struct EmaParams {
  float* slab;             // the averages, a slab in the plan's layout (16-byte aligned)
  EmaState* state;
  float decay;             // fp32(decay)
  int32_t num_updates;     // 1: d = min(decay, (1 + n) / (10 + n))
};

// Per-tensor learning-rate multipliers (gaccum_plan_set_lr_multipliers).  Every plan has the table (1.0 unless set), so
// no kernel is specialised on it: each apply kernel reads mult[t] once per tile and uses the tile's rate (tile_rate).
struct LrMultParams {
  const float* mult;       // num_tensors
};

// gaccum_window_weight_state (gaccum.h): caller-owned device memory.  The producer adds each micro-batch's weight into
// `weight`; every apply launch of a weighted plan divides by it, then stores last_weight = W and weight = +0.
struct WindowWeightState {
  float weight;            // W: the running window's total weight
  float last_weight;       // W of the last apply launch
  float reserved[2];
};
static_assert(sizeof(WindowWeightState) == 16, "gaccum_window_weight_state is 16 bytes");

// Per-window normalisation (gaccum_plan_set_window_weight): c = a'/W in place of a'/N.  state == NULL: divide by N.
struct WindowWeightParams {
  WindowWeightState* state;
};

// gaccum_schedule_state (gaccum.h): caller-owned device memory, written by gaccum_schedule_init and afterwards only by
// the launches of a device-scheduled plan
struct ScheduleState {
  long long global_step;        // the pre-increment step of the next launch
  long long num_train_steps;
  long long num_warmup_steps;
  float init_lr;                // fp32(init_lr)
  float end_lr;                 // 0
  float power;                  // 1
  float beta1_power, beta2_power;   // GACCUM_ADAM, GACCUM_LAMB without loss scaling (else the loss-scaling block's)
  int32_t refused;              // 1 once a launch found global_step selecting the other branch: every launch is a no-op
};
static_assert(sizeof(ScheduleState) == 48, "gaccum_schedule_state is 48 bytes");

// The device schedule (gaccum_plan_set_device_schedule).  state == NULL: the host's lr and beta powers (Scalars).  A
// launch-uniform branch, not a template flag: no kernel is specialised on it.
struct ScheduleParams {
  ScheduleState* state;
  int32_t accum_n;         // N: the launch checks that global_step selects its branch
};

// Per-tensor norms of the apply step (gaccum_plan_set_tensor_norms).  out == NULL: off.  A launch-uniform branch, not a
// template flag: no kernel is specialised on it.  The reduction is deterministic without atomics on the sums:
//   1. the apply kernels store, for every tile, column (gradient, weight, update) and warp of the 256 threads that walked
//      the tile, the warp's fp64 total of its threads' fp32 partials (tile_part; plain stores, each slot written once);
//   2. a chunk of up to kNormChunk consecutive tiles of one tensor is summed by one warp, tile by tile and warp by warp
//      in that order (chunk_part), once all its tiles are written;
//   3. the tensor's chunks are summed in chunk order by the warp that finishes its last chunk (a counter per tensor),
//      and out[3t + k] = sqrtf(fp32(sum)).
// Every order is fixed by the tile table alone, so the values do not depend on which CTA, group or path took a tile.
constexpr int kNormCols = 3;                     // gradient, weight, update
constexpr int kNormWarps = kThreads / 32;        // warps of the 256 threads that walk one tile
constexpr int kNormChunk = 32;                   // tiles per chunk: one per lane of the summing warp
struct NormParams {
  float* out;                  // num_tensors x 3, caller-owned
  double* tile_part;           // num_tiles x kNormCols x kNormWarps
  double* chunk_part;          // num_chunks x kNormCols
  const int32_t* tile_begin;   // num_tensors + 1: tensor t owns tiles [tile_begin[t], tile_begin[t + 1])
  const int32_t* chunk_begin;  // num_tensors + 1: ... and chunks [chunk_begin[t], chunk_begin[t + 1])
  const int32_t* chunk_tensor; // num_chunks
  unsigned int* chunk_done;    // num_chunks: apply_kernel's tiles of the chunk that are through (0 between launches)
  unsigned int* tensor_done;   // num_tensors: chunks of the tensor that are summed (0 between launches)
  int32_t num_chunks;
};

// A learning-rate table of a device-scheduled plan (gaccum_plan_set_lr_table): caller-owned device memory, read at
// launch time.  table == NULL: schedule_lr.  A launch-uniform branch in sched_load, not a template flag.
struct LrTableParams {
  const float* table;
  int64_t length;          // >= 1
};

// Deferred reset of the accumulators (gaccum_plan_set_deferred_reset).  accum_zero == NULL: every apply stores a = +0, as
// the reference does.  Otherwise no apply stores into the accumulator slab: its commit sets the plan's word *accum_zero to
// 1, which makes the accumulators logically +0 and the slab's contents unspecified.  The first accumulate of a window
// (which does not read a) then stores +0 + G where there is a gradient and, while the word is 1, +0 where there is none;
// the last of its CTAs clears the word.  A launch-uniform branch, not a template flag: no kernel is specialised on it.
struct DeferredResetParams {
  unsigned int* accum_zero;
};

// Every kernel's parameter block.  Each feature's parameters follow those of the features before it, so adding them
// moved no member an existing kernel reads.
template <int CAP>
struct KernelParams {
  const TileDesc* tiles;
  int32_t num_tiles;
  float* accum;
  float* m;
  float* v;
  float* stats;       // gaccum_stats
  unsigned long long* barrier;  // apply_clip_kernel: monotonic arrival counter of the consumers' grid barrier
  struct LaunchCounters* counters;  // apply_clip_kernel: two sets of per-launch counters (tickets, pool length, norm accumulator)
  unsigned int* done;   // apply_kernel, scheduled accumulate_kernel: CTAs of the launch that are through (0 between launches)
#ifdef GACCUM_EXPERIMENTS
  unsigned long long* debug;  // 16 words per CTA: 4 timestamps (ns) + wait-cycle counters (tools/cta_timeline.py)
#endif
  Scalars sc;
  PtrTable<CAP> tab;
  LossScaleParams ls;   // loss-scaled modes (kLsClip, kLsNoClip) only
  HalfParams half;      // kernels with H = true only
  LambParams lamb;      // lamb_apply_kernel only
  EmaParams ema;        // kernels with EMA = true only
  LrMultParams lrm;     // apply kernels only
  WindowWeightParams ww;  // apply kernels only
  ScheduleParams sched;   // every kernel
  NormParams norms;       // apply kernels only
  LrTableParams lrt;      // device-scheduled launches only
  DeferredResetParams dr; // apply kernels and the first accumulate of a window only
};
static_assert(sizeof(KernelParams<1920>) <= 32764, "kernel parameters must fit the 32 KB limit");

// optimization.py:29-54 exactly as gaccum_learning_rate evaluates it on the host: polynomial decay (end 0, power 1) of
// min(g, T) over T, then, with a warm-up, (1 - is_warmup) * lr + is_warmup * (init_lr * (int32(g) / int32(W))).  One
// correctly rounded fp32 op per TF op; int64 -> fp32 and int32 -> fp32 conversions round to nearest.
__device__ __forceinline__ float schedule_lr(const float init_lr, const long long T, const long long W, const long long g) {
  float gs = __ll2float_rn(g);
  const float ds = __ll2float_rn(T);
  if (gs > ds) gs = ds;
  const float p = __fdiv_rn(gs, ds);
  float lr = __fmul_rn(init_lr, __fsub_rn(1.0f, p));
  if (W != 0) {
    const int gi = (int)g, wi = (int)W;
    const float pct = __fdiv_rn(__int2float_rn(gi), __int2float_rn(wi));
    const float wlr = __fmul_rn(init_lr, pct);
    const float isw = gi < wi ? 1.0f : 0.0f;
    lr = __fadd_rn(__fmul_rn(__fsub_rn(1.0f, isw), lr), __fmul_rn(isw, wlr));
  }
  return lr;
}
// The learning rate of a device-scheduled launch (a LaunchStep) at the block's step g -- table[min(g, length - 1)] with
// a learning-rate table (g >= 0: gaccum_schedule_init keeps it so; a 64-bit index, untouched by the int32 wrap), else
// schedule_lr -- the beta powers as the block holds them, and whether the launch may run: g selects its branch (apply),
// no earlier launch was refused, and a first accumulate (from_zero), which does not read the accumulators, follows a
// step that applied and left them at +0 ((int32)(g - 1) % N == 0) -- else it would overwrite that step's gradients
template <typename Step>
__device__ __forceinline__ void sched_load(const ScheduleParams& sp, const LrTableParams& lt, const bool apply,
                                           const bool from_zero, Step& sl) {
  const ScheduleState* st = sp.state;
  const long long g = __ldcg(&st->global_step);
  if (lt.table)                                    // launch-uniform
    sl.lr = __ldcg(&lt.table[g < lt.length ? g : lt.length - 1]);
  else
    sl.lr = schedule_lr(__ldcg(&st->init_lr), __ldcg(&st->num_train_steps), __ldcg(&st->num_warmup_steps), g);
  sl.b1p = __ldcg(&st->beta1_power);
  sl.b2p = __ldcg(&st->beta2_power);
  sl.ok = __ldcg(&st->refused) == 0 && ((((int)g % sp.accum_n) == 0) == apply)    // gaccum_is_apply_step
          && (!from_zero || ((int)(g - 1) % sp.accum_n) == 0);
}
// The next step, and (betas) TF1's beta powers advanced with one fp32 multiply each, as after an applied window.  Only
// this commit writes the block, so it still holds what the launch found.
__device__ __forceinline__ void sched_finish(const ScheduleParams& sp, const bool betas, const float b1, const float b2) {
  ScheduleState* st = sp.state;
  st->global_step = __ldcg(&st->global_step) + 1;
  if (betas) {
    st->beta1_power = __fmul_rn(__ldcg(&st->beta1_power), b1);
    st->beta2_power = __fmul_rn(__ldcg(&st->beta2_power), b2);
  }
}
// A launch whose branch global_step does not select (a captured graph whose start is not a window start, or a window
// that straddles the int32 wrap of global_step), or a first accumulate that does not follow an apply, changes nothing;
// block 0 marks the schedule refused, so every later launch is a no-op too and the host can report it.
__device__ __forceinline__ void sched_refuse(const ScheduleParams& sp) {
  if (blockIdx.x == 0 && threadIdx.x == 0) sp.state->refused = 1;
}

// What every CTA of an EMA launch derives from the state as the launch finds it (TF1 ExponentialMovingAverage, one
// correctly rounded fp32 op per TF op): d = fp32(decay), in num_updates mode d = min(d, (1 + fp32(n)) / (10 + fp32(n)));
// c = 1 - d (assign_moving_average's `1.0 - decay`)
struct EmaLaunch {
  long long n;
  float d, c;
};
__device__ __forceinline__ void ema_load(const EmaParams& ep, EmaLaunch& el) {
  const long long n = __ldcg(&ep.state->num_updates);
  float d = ep.decay;
  if (ep.num_updates) {
    const float nf = (float)n;                                         // round to nearest, as TF's cast
    const float w = __fdiv_rn(__fadd_rn(1.0f, nf), __fadd_rn(10.0f, nf));
    d = w < d ? w : d;
  }
  el.n = n;
  el.d = d;
  el.c = __fsub_rn(1.0f, d);
}
// one averaged window: n + 1 windows averaged, the last with decay d
__device__ __forceinline__ void ema_finish(const EmaParams& ep, const EmaLaunch& el) {
  EmaState s;
  s.num_updates = el.n + 1;
  s.decay = el.d;
  s.reserved = 0.f;
  *ep.state = s;
}
// e = e - (e - p) * c: assign_sub of the update delta; p is the value the apply just stored
__device__ __forceinline__ float ema_elem(float e, float p, float c) { return __fsub_rn(e, __fmul_rn(__fsub_rn(e, p), c)); }
__device__ __forceinline__ float4 ema_vec(const float4 e, const float4 p, float c) {
  return make_float4(ema_elem(e.x, p.x, c), ema_elem(e.y, p.y, c), ema_elem(e.z, p.z, c), ema_elem(e.w, p.w, c));
}

// ---------------------------------------------------------------------------------------------
// memory helpers: G is read exactly once -> streaming (evict-first) loads; zeroing the
// accumulator is a streaming store.  a' must survive in L2 from pass 1 to pass 2, so it is
// tagged evict_last while everything that is touched once is tagged evict-first.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float4 ld_stream(const float4* p) { return __ldcs(p); }
__device__ __forceinline__ float ld_stream(const float* p) { return __ldcs(p); }
__device__ __forceinline__ uint64_t policy_evict_last() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ uint64_t policy_evict_first() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ float4 ld_policy(const float4* p, uint64_t pol) {
  float4 v;
  asm volatile("ld.global.L2::cache_hint.v4.f32 {%0,%1,%2,%3}, [%4], %5;"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p), "l"(pol) : "memory");
  return v;
}
__device__ __forceinline__ void st_policy(float4* p, const float4 v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.v4.f32 [%0], {%1,%2,%3,%4}, %5;"
               :: "l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w), "l"(pol) : "memory");
}
// Drop the 128-byte L2 line at p (128-byte aligned) without writing it back: its contents become unspecified.  For dead
// accumulator lines of a deferred-reset apply (DeferredResetParams), which would otherwise be written back dirty.
__device__ __forceinline__ void discard_line(const void* p) {
  asm volatile("discard.global.L2 [%0], 128;" :: "l"(p) : "memory");
}

template <int CAP>
__device__ __forceinline__ const float* grad_ptr(const PtrTable<CAP>& tab, const TileDesc& d) {
  if constexpr (CAP == 0) {
    return tab.g ? tab.g + (size_t)d.soff32 * kSlabAlign : nullptr;
  } else {
    const float* b = tab.g[d.tensor_flags & 0x7fffffffu];
    return b ? b + d.toff : nullptr;
  }
}
template <int CAP>
__device__ __forceinline__ float* param_ptr(const PtrTable<CAP>& tab, const TileDesc& d) {
  if constexpr (CAP == 0) {
    return tab.p + (size_t)d.soff32 * kSlabAlign;
  } else {
    return tab.p[d.tensor_flags & 0x7fffffffu] + d.toff;
  }
}
__device__ __forceinline__ bool aligned16(const void* p) { return ((uintptr_t)p & 15u) == 0; }
__device__ __forceinline__ bool aligned8(const void* p) { return ((uintptr_t)p & 7u) == 0; }

// ---- 16-bit models: widening is exact; narrowing rounds to nearest-even (cvt.rn), as torch's .to(dtype) does ----
__device__ __forceinline__ float h2f(uint16_t x, bool bf16) {
  return bf16 ? __uint_as_float((uint32_t)x << 16) : __half2float(__ushort_as_half(x));
}
__device__ __forceinline__ uint32_t f2h(float x, bool bf16) {
  return bf16 ? (uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(x)) : (uint32_t)__half_as_ushort(__float2half_rn(x));
}
__device__ __forceinline__ float4 h2f4(const uint2 r, bool bf16) {   // 4 elements, the first in the low half of r.x
  return make_float4(h2f((uint16_t)r.x, bf16), h2f((uint16_t)(r.x >> 16), bf16), h2f((uint16_t)r.y, bf16),
                     h2f((uint16_t)(r.y >> 16), bf16));
}
// the model copy of 4 master weights at elements 4i..4i+3: one 8-byte store if the tensor is 8-byte aligned
__device__ __forceinline__ void store_model4(uint16_t* q, uint32_t i, const float4 p, bool bf16) {
  if (aligned8(q)) {
    __stcs(reinterpret_cast<uint2*>(q) + i, make_uint2(f2h(p.x, bf16) | (f2h(p.y, bf16) << 16), f2h(p.z, bf16) | (f2h(p.w, bf16) << 16)));
  } else {
    q[4 * i] = (uint16_t)f2h(p.x, bf16); q[4 * i + 1] = (uint16_t)f2h(p.y, bf16);
    q[4 * i + 2] = (uint16_t)f2h(p.z, bf16); q[4 * i + 3] = (uint16_t)f2h(p.w, bf16);
  }
}

// The gradient stream of one tile, widened to fp32 on load.  H: bf16 / fp16, the vector path reads 4 x 16 bit (8 B).
// A default-constructed Grad is "no gradient" (g == nullptr).
template <bool H> struct Grad;
template <>
struct Grad<false> {
  const float* g = nullptr;
  __device__ __forceinline__ Grad() {}
  template <int CAP>
  __device__ __forceinline__ Grad(const KernelParams<CAP>& prm, const TileDesc& d) : g(grad_ptr(prm.tab, d)) {}
  __device__ __forceinline__ bool vec_ok() const { return aligned16(g); }
  __device__ __forceinline__ float4 vec(uint32_t i) const { return ld_stream(reinterpret_cast<const float4*>(g) + i); }
  __device__ __forceinline__ float elem(uint32_t i) const { return ld_stream(g + i); }
  // the G half of a pass-1 ring slot
  __device__ __forceinline__ float4 slot(const float4* s, uint32_t i) const { return s[i]; }
};
template <>
struct Grad<true> {
  const uint16_t* g = nullptr;
  bool bf16 = false;
  __device__ __forceinline__ Grad() {}
  template <int CAP>
  __device__ __forceinline__ Grad(const KernelParams<CAP>& prm, const TileDesc& d) : bf16(prm.half.bf16 != 0) {
    const uint16_t* b = reinterpret_cast<const uint16_t*>(prm.tab.g[d.tensor_flags & 0x7fffffffu]);
    g = b ? b + d.toff : nullptr;
  }
  __device__ __forceinline__ bool vec_ok() const { return aligned8(g); }
  __device__ __forceinline__ float4 vec(uint32_t i) const { return h2f4(__ldcs(reinterpret_cast<const uint2*>(g) + i), bf16); }
  __device__ __forceinline__ float elem(uint32_t i) const { return h2f(__ldcs(g + i), bf16); }
  __device__ __forceinline__ float4 slot(const float4* s, uint32_t i) const { return h2f4(reinterpret_cast<const uint2*>(s)[i], bf16); }
};

// The fp32 weights the update reads and writes: the parameters themselves, or (H) the master slab
template <bool H, int CAP>
__device__ __forceinline__ float* update_ptr(const KernelParams<CAP>& prm, const TileDesc& d) {
  if constexpr (H) return prm.half.master + (size_t)d.soff32 * kSlabAlign;
  else return param_ptr(prm.tab, d);
}
// H: the model copy of the tile (16-bit)
template <int CAP>
__device__ __forceinline__ uint16_t* model_ptr(const KernelParams<CAP>& prm, const TileDesc& d) {
  return reinterpret_cast<uint16_t*>(prm.tab.p[d.tensor_flags & 0x7fffffffu]) + d.toff;
}

// ---------------------------------------------------------------------------------------------
// per-element math, one rounding per reference op
// ---------------------------------------------------------------------------------------------
// optimization.py:83  (1.0*a)/N  -- the multiply by 1.0 is exact.  When N is a power of two, 1/N is
// exact and a * (1/N) is the same correctly rounded real number as a / N (bit-identical, subnormals
// included), which saves a ~12-instruction IEEE division per element; otherwise divide.
__device__ __forceinline__ float normalize(float a, float nf, float inv_nf) {
  return inv_nf != 0.f ? __fmul_rn(a, inv_nf) : __fdiv_rn(a, nf);
}

// The divisor D of c = (1.0*a')/D, as normalize() takes it: fp32(N) from Scalars, or a weighted plan's window weight W.
// The functions that normalise take either (Scalars or Divisor: both have nf and inv_nf).
struct Divisor {
  float nf;       // D
  float inv_nf;   // 1/D when D is a normal power of two (exact), else 0 -> the kernels divide
};
// W as a divisor: the rule make_scalars applies to N, so a / W is always the correctly rounded quotient.  A W that is
// zero, negative, subnormal or not finite is divided by as it is (IEEE results, as a NaN gradient propagates).
__device__ __forceinline__ Divisor weight_divisor(float W) {
  const uint32_t bits = __float_as_uint(W), e = (bits >> 23) & 0xffu;
  return Divisor{W, ((bits & 0x007fffffu) == 0u && e != 0u && e != 0xffu) ? __fdiv_rn(1.0f, W) : 0.f};
}
// The divisor of one apply launch: W as the state holds it when the launch starts (weighted plans), else N
template <typename KP>
__device__ __forceinline__ Divisor launch_divisor(const KP& prm) {
  return prm.ww.state ? weight_divisor(__ldcg(&prm.ww.state->weight)) : Divisor{prm.sc.nf, prm.sc.inv_nf};
}
// Once every CTA of the launch has read W: record it, and start the next window at +0 (applied or skipped alike)
__device__ __forceinline__ void window_finish(WindowWeightState* st, float W) {
  st->last_weight = W;
  st->weight = 0.f;
}

// rate: the tile's learning rate lr_t (VARIANT 0) or alpha_t (VARIANT 1) the update uses (tile_rate)
template <int VARIANT>
__device__ __forceinline__ void adam_elem(float c, float& p, float& m, float& v, bool decay,
                                          const Scalars& sc, const float& rate) {
  if constexpr (VARIANT == 0) {
    // optimization.py:151-171
    const float m2 = __fadd_rn(__fmul_rn(sc.b1, m), __fmul_rn(sc.omb1, c));
    const float v2 = __fadd_rn(__fmul_rn(sc.b2, v), __fmul_rn(sc.omb2, __fmul_rn(c, c)));
    float u = __fdiv_rn(m2, __fadd_rn(__fsqrt_rn(v2), sc.eps));
    if (decay) u = __fadd_rn(u, __fmul_rn(sc.wd, p));
    p = __fsub_rn(p, __fmul_rn(rate, u));
    m = m2;
    v = v2;
  } else {
    // TF1 ApplyAdam: m += (g-m)(1-b1); v += (g*g-v)(1-b2); var -= (m*alpha)/(sqrt(v)+eps)
    const float m2 = __fadd_rn(m, __fmul_rn(__fsub_rn(c, m), sc.omb1));
    const float v2 = __fadd_rn(v, __fmul_rn(__fsub_rn(__fmul_rn(c, c), v), sc.omb2));
    p = __fsub_rn(p, __fdiv_rn(__fmul_rn(m2, rate), __fadd_rn(__fsqrt_rn(v2), sc.eps)));
    m = m2;
    v = v2;
  }
}
// The tile's rate for tensor multiplier `mult`: lr_t = lr * mult, one correctly rounded multiply; GACCUM_ADAM:
// alpha_t = (lr_t * sqrt(1 - b2^t)) / (1 - b1^t), with bc2 and bc1 those two bias-correction terms -- TF1 ApplyAdam's
// alpha, one rounding per op, when mult == 1.
template <int VARIANT>
__device__ __forceinline__ float tile_rate(const float lr, const float mult, const float bc2, const float bc1) {
  const float lr_t = __fmul_rn(lr, mult);
  if constexpr (VARIANT == 0) return lr_t;
  else return __fdiv_rn(__fmul_rn(lr_t, bc2), bc1);
}
__device__ __forceinline__ float tensor_mult(const LrMultParams& lrm, const TileDesc& d) {
  return __ldg(lrm.mult + (d.tensor_flags & 0x7fffffffu));
}

// optimization.py:83-85: c = a/D (dv: N, or the window weight W), times the clip scale s if `scaled` (never a multiply
// by 1: it could change a NaN's payload), then one Adam step of p, m, v with `rate` (tile_rate)
template <int VARIANT, typename D>
__device__ __forceinline__ void update_elem(float a, bool scaled, float s, float& p, float& m, float& v, bool decay,
                                            const Scalars& sc, const float& rate, const D& dv) {
  float c = normalize(a, dv.nf, dv.inv_nf);
  if (scaled) c = __fmul_rn(c, s);
  adam_elem<VARIANT>(c, p, m, v, decay, sc, rate);
}
template <int VARIANT, typename D>
__device__ __forceinline__ void update_vec(const float4 a, bool scaled, float s, float4& p, float4& m, float4& v, bool decay,
                                           const Scalars& sc, const float& rate, const D& dv) {
  update_elem<VARIANT>(a.x, scaled, s, p.x, m.x, v.x, decay, sc, rate, dv);
  update_elem<VARIANT>(a.y, scaled, s, p.y, m.y, v.y, decay, sc, rate, dv);
  update_elem<VARIANT>(a.z, scaled, s, p.z, m.z, v.z, decay, sc, rate, dv);
  update_elem<VARIANT>(a.w, scaled, s, p.w, m.w, v.w, decay, sc, rate, dv);
}

__device__ __forceinline__ float4 add_rn(const float4 a, const float4 b) {
  return make_float4(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y), __fadd_rn(a.z, b.z), __fadd_rn(a.w, b.w));
}
// per-tensor norms (NormParams): a thread's fp32 partial of one tile's column: acc + x^2, and acc + (p - q)^2 with the fp32 difference
__device__ __forceinline__ float sq_acc(float acc, float x) { return fmaf(x, x, acc); }
__device__ __forceinline__ float sq_acc(float acc, const float4 x) {
  return sq_acc(sq_acc(sq_acc(sq_acc(acc, x.x), x.y), x.z), x.w);
}
__device__ __forceinline__ float diff_sq_acc(float acc, float p, float q) {
  const float d = __fsub_rn(p, q);
  return fmaf(d, d, acc);
}
// acc + (x/D)^2: one element of a thread's fp32 partial of the global norm
template <typename D>
__device__ __forceinline__ float add_sq(float acc, float x, const D& dv) {
  const float n = normalize(x, dv.nf, dv.inv_nf);
  return fmaf(n, n, acc);
}
template <typename D>
__device__ __forceinline__ float add_sq(float acc, const float4 x, const D& dv) {
  return add_sq(add_sq(add_sq(add_sq(acc, x.x, dv), x.y, dv), x.z, dv), x.w, dv);
}

// Loss scaling: the accumulators hold sums of S*g.  c = ((1.0*a')/D) * (1/S), two correctly rounded ops; S is a power of
// two, so the multiply is exact wherever c is a normal number.  Pass 1 also notes any non-finite element of a'.
template <typename D>
__device__ __forceinline__ float unscale(float a, float inv_s, const D& dv) {
  return __fmul_rn(normalize(a, dv.nf, dv.inv_nf), inv_s);
}
template <int MODE, typename D>
__device__ __forceinline__ float ls_pass1(float acc, float x, float inv_s, bool& bad, const D& dv) {
  bad |= !(fabsf(x) <= 3.402823466e38f);
  if constexpr (MODE == kLsClip) {
    const float c = unscale(x, inv_s, dv);
    acc = fmaf(c, c, acc);
  }
  return acc;
}
template <int MODE, typename D>
__device__ __forceinline__ float ls_pass1(float acc, const float4 x, float inv_s, bool& bad, const D& dv) {
  return ls_pass1<MODE>(ls_pass1<MODE>(ls_pass1<MODE>(ls_pass1<MODE>(acc, x.x, inv_s, bad, dv), x.y, inv_s, bad, dv), x.z, inv_s, bad, dv),
                        x.w, inv_s, bad, dv);
}
// c of one element of a' in the cooperative kernels: (1.0*a')/D, unscaled by 1/S under loss scaling, times the clip
// scale s when clipping
template <int MODE, typename D>
__device__ __forceinline__ float mode_c(float a, float s, float inv_s, const D& dv) {
  if constexpr (MODE == kNoClip) return normalize(a, dv.nf, dv.inv_nf);
  else if constexpr (MODE == kClip) return __fmul_rn(normalize(a, dv.nf, dv.inv_nf), s);
  else if constexpr (MODE == kLsClip) return __fmul_rn(unscale(a, inv_s, dv), s);
  else return unscale(a, inv_s, dv);
}
// pass 2 of the clip kernel on 4 elements: c of a', then one Adam step each.  A function of its own: written out at the
// call site, nvcc schedules the AdamWeightDecay instantiations differently (more instructions, different registers).
template <int VARIANT, int MODE>
__device__ __forceinline__ void adam_vec(const float4 a, float s, float inv_s, float4& p, float4& m, float4& v, bool decay,
                                         const Scalars& sc, const float& rate, const Divisor& dv) {
  adam_elem<VARIANT>(mode_c<MODE>(a.x, s, inv_s, dv), p.x, m.x, v.x, decay, sc, rate);
  adam_elem<VARIANT>(mode_c<MODE>(a.y, s, inv_s, dv), p.y, m.y, v.y, decay, sc, rate);
  adam_elem<VARIANT>(mode_c<MODE>(a.z, s, inv_s, dv), p.z, m.z, v.z, decay, sc, rate);
  adam_elem<VARIANT>(mode_c<MODE>(a.w, s, inv_s, dv), p.w, m.w, v.w, decay, sc, rate);
}

// tf.clip_by_global_norm (TF 1.15): scale = clip * min(1/gn, 1/clip) + (gn - gn)
__device__ __forceinline__ float clip_scale(float gn, float clip) {
  const float inv = __fdiv_rn(1.0f, gn);
  const float invc = __fdiv_rn(1.0f, clip);
  float mn = inv < invc ? inv : invc;
  if (inv != inv) mn = inv;
  return __fadd_rn(__fmul_rn(clip, mn), __fsub_rn(gn, gn));
}

// ---- per-tensor norms (NormParams) ----------------------------------------------------------------------------
// warp total of a per-thread double, fixed butterfly order (lane 0's value is the one every caller uses)
__device__ __forceinline__ double warp_sum(double w) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) w += __shfl_xor_sync(0xffffffffu, w, o);
  return w;
}
// the whole warp: its fp64 total of the threads' partials `part` of (tile, col), stored by lane 0
__device__ __forceinline__ void norm_store(const NormParams& np, const int tile, const int col, const int warp, const float part) {
  const double w = warp_sum((double)part);
  if ((threadIdx.x & 31) == 0) np.tile_part[((size_t)tile * kNormCols + col) * kNormWarps + warp] = w;
}
// The whole warp, once every tile of chunk c is stored: the chunk's sums (lane l takes tile l of the chunk and adds its
// warps' partials in order; then the butterfly), and, if this is the tensor's last chunk to be summed, the tensor's norms
// from its chunks in chunk order.  The finishing warp resets the tensor's counter for the next launch.
__device__ __noinline__ void norm_chunk(const NormParams& np, const int c) {
  const int lane = (int)threadIdx.x & 31;
  const int t = __ldg(np.chunk_tensor + c);
  const int cb = __ldg(np.chunk_begin + t), ce = __ldg(np.chunk_begin + t + 1);
  const int tile = __ldg(np.tile_begin + t) + (c - cb) * kNormChunk + lane;
  double s[kNormCols] = {0.0, 0.0, 0.0};
  if (tile < __ldg(np.tile_begin + t + 1)) {
    const double* tp = np.tile_part + (size_t)tile * kNormCols * kNormWarps;
#pragma unroll
    for (int k = 0; k < kNormCols; ++k)
#pragma unroll
      for (int w = 0; w < kNormWarps; ++w) s[k] += __ldcg(tp + k * kNormWarps + w);
  }
#pragma unroll
  for (int k = 0; k < kNormCols; ++k) s[k] = warp_sum(s[k]);
  unsigned int last = 0;
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < kNormCols; ++k) np.chunk_part[(size_t)c * kNormCols + k] = s[k];
    __threadfence();
    last = atomicAdd(np.tensor_done + t, 1u) == (unsigned int)(ce - cb - 1);
  }
  if (!__shfl_sync(0xffffffffu, last, 0)) return;
  __threadfence();
  double r[kNormCols] = {0.0, 0.0, 0.0};
  for (int k = cb + lane; k < ce; k += 32) {
#pragma unroll
    for (int j = 0; j < kNormCols; ++j) r[j] += __ldcg(np.chunk_part + (size_t)k * kNormCols + j);
  }
#pragma unroll
  for (int j = 0; j < kNormCols; ++j) r[j] = warp_sum(r[j]);
  if (lane == 0) {
#pragma unroll
    for (int j = 0; j < kNormCols; ++j) np.out[(size_t)t * kNormCols + j] = __fsqrt_rn((float)r[j]);
    np.tensor_done[t] = 0u;
  }
}
// Every warp of a cooperative launch, past a grid barrier that follows the last tile_part store: every chunk, `gw` the
// warp's index among `nw`
__device__ __forceinline__ void norm_finish_all(const NormParams& np, const int gw, const int nw) {
  for (int c = gw; c < np.num_chunks; c += nw) norm_chunk(np, c);
}
// apply_kernel, one tile per CTA, after every warp stored the tile's partials: thread 0 counts the tile into its chunk;
// the CTA that completes the chunk sums it with warp 0
__device__ __forceinline__ void norm_arrive_tile(const NormParams& np, const TileDesc& d, const int tile) {
  __shared__ int s_chunk;
  __syncthreads();
  if (threadIdx.x == 0) {
    const int t = (int)(d.tensor_flags & 0x7fffffffu);
    const int tb = __ldg(np.tile_begin + t), te = __ldg(np.tile_begin + t + 1);
    const int j = (tile - tb) / kNormChunk;
    const int c = __ldg(np.chunk_begin + t) + j;
    const int n = min(kNormChunk, te - tb - j * kNormChunk);
    __threadfence();
    const bool last = atomicAdd(np.chunk_done + c, 1u) == (unsigned int)(n - 1);
    if (last) np.chunk_done[c] = 0u;
    s_chunk = last ? c : -1;
  }
  __syncthreads();
  if (s_chunk >= 0 && threadIdx.x < 32) {
    __threadfence();
    norm_chunk(np, s_chunk);
  }
}

// ---------------------------------------------------------------------------------------------
// One tile as every per-tile function walks it: thread `tid` owns the float4 vectors tid and tid + kThreads that are
// below `nvec`, then at most one of the < 4 trailing elements.  nvec == 0 means the tile cannot take the vector path
// (a view that is not 16-byte aligned, or fewer than 4 elements): `elem` then covers the whole tile, kThreads apart.
// All of a thread's vector loads are issued before its first store; `loaded` runs between the two.
// ---------------------------------------------------------------------------------------------
template <typename Load, typename Loaded, typename Vec, typename Elem>
__device__ __forceinline__ void walk_tile(const uint32_t len, const uint32_t nvec, const uint32_t tid, Load&& load,
                                          Loaded&& loaded, Vec&& vec, Elem&& elem) {
#pragma unroll
  for (int u = 0; u < kUnroll; ++u) {
    const uint32_t i = u * kThreads + tid;
    if (i < nvec) load(u, i);
  }
  loaded();
#pragma unroll
  for (int u = 0; u < kUnroll; ++u) {
    const uint32_t i = u * kThreads + tid;
    if (i < nvec) vec(u, i);
  }
  for (uint32_t i = (nvec << 2) + tid; i < len; i += kThreads) elem(i);
}

// ---------------------------------------------------------------------------------------------
// accumulate: a += G                                                   optimization.py:81,93
// FROM_ZERO: the first accumulate of a window.  The apply that ended the previous window left every accumulator at
// +0.0 (optimization.py:78,86-87), so a is not loaded and a = +0 + G is stored (8 instead of 12 B/elem).  The add is
// kept: it turns a gradient of -0.0 into +0.0, as assign_add onto a zero does, and a NaN comes out as a += G gives it.
// zero (FROM_ZERO, deferred reset only): the slab holds no zeros (DeferredResetParams), so a tile without a gradient
// stores them.
// ---------------------------------------------------------------------------------------------
template <bool FROM_ZERO, bool H, int CAP>
__device__ __forceinline__ void accumulate_tile(const TileDesc d, const KernelParams<CAP>& prm, const bool zero) {
  const Grad<H> g(prm, d);
  float* __restrict__ a = prm.accum + (size_t)d.soff32 * kSlabAlign;
  float4* a4 = reinterpret_cast<float4*>(a);
  if (g.g == nullptr) {         // optimization.py:132 -- tensors without a gradient are skipped
    if (FROM_ZERO && zero) {    // the slab is 16-byte aligned at every tile
      walk_tile(d.len, d.len >> 2, threadIdx.x, [](int, uint32_t) {}, [] {},
                [&](int, uint32_t i) { a4[i] = make_float4(0.f, 0.f, 0.f, 0.f); }, [&](uint32_t i) { a[i] = 0.f; });
    }
    return;
  }
  float4 vg[kUnroll], va[kUnroll];
  walk_tile(d.len, g.vec_ok() ? d.len >> 2 : 0u, threadIdx.x,
            [&](int u, uint32_t i) {
              vg[u] = g.vec(i);
              if constexpr (FROM_ZERO) va[u] = make_float4(0.f, 0.f, 0.f, 0.f); else va[u] = a4[i];
            },
            [] {},
            [&](int u, uint32_t i) { a4[i] = add_rn(va[u], vg[u]); },
            [&](uint32_t i) { a[i] = __fadd_rn(FROM_ZERO ? 0.f : a[i], g.elem(i)); });
}

// ---------------------------------------------------------------------------------------------
// One launch's step: what it reads from the device state blocks when it starts (launch_begin) and what it writes back
// when it ends (launch_commit).
// ---------------------------------------------------------------------------------------------
// loss scaling: the state as this launch finds it
__device__ __forceinline__ void ls_load(const LossScaleState* st, LossScaleState& s) {
  s.scale = __ldcg(&st->scale);
  s.good_windows = __ldcg(&st->good_windows);
  s.skipped_windows = __ldcg(&st->skipped_windows);
  s.beta1_power = __ldcg(&st->beta1_power);
  s.beta2_power = __ldcg(&st->beta2_power);
}
// TF 2 DynamicLossScale, counted in windows (gaccum.h, gaccum_loss_scale_config); BETAS: the optimizer keeps TF1's beta
// powers, advanced on applied windows only
template <bool BETAS>
__device__ __forceinline__ void ls_finish(const LossScaleParams& ls, const LossScaleState& s_ls, const bool skip,
                                          const float b1, const float b2) {
  LossScaleState* out = ls.state;
  const float S = s_ls.scale;
  if (skip) {
    const float down = __fdiv_rn(S, ls.multiplier);   // exact: both are powers of two
    out->scale = down < 1.0f ? 1.0f : down;
    out->good_windows = 0;
    out->skipped_windows = s_ls.skipped_windows + 1u;
    out->last_skipped = 1;
  } else {
    const int32_t good = s_ls.good_windows + 1;
    if (good >= ls.growth_interval) {
      const float up = __fmul_rn(S, ls.multiplier);
      if (fabsf(up) <= 3.402823466e38f) out->scale = up;
      out->good_windows = 0;
    } else {
      out->good_windows = good;
    }
    out->last_skipped = 0;
    if constexpr (BETAS) {                            // TF1 AdamOptimizer._finish, applied windows only
      out->beta1_power = __fmul_rn(s_ls.beta1_power, b1);
      out->beta2_power = __fmul_rn(s_ls.beta2_power, b2);
    }
  }
}

// The VARIANT of launch_begin and launch_commit: the optimizer of an apply launch (gaccum.h: 0 GACCUM_ADAM_WEIGHT_DECAY,
// 1 GACCUM_ADAM, 2 GACCUM_LAMB), or kAccumulate
constexpr int kLamb = 2;
constexpr int kAccumulate = -1;
// GACCUM_ADAM and GACCUM_LAMB keep TF1's beta powers: every applied window advances them
__host__ __device__ constexpr bool keeps_beta_powers(int variant) { return variant == 1 || variant == kLamb; }

// The part of a LaunchStep that only EMA kernels have: an empty base otherwise, so no kernel's shared memory grows
template <bool EMA> struct StepEma {};
template <> struct StepEma<true> { EmaLaunch ema; };
// The step as one launch finds it.  A loss-scaled launch also finds the loss-scaling state, which it keeps in a shared
// object of its own: held in the same object, the packed Adam kLsClip clip-apply spills 12 more bytes per thread.
template <bool EMA = false>
struct LaunchStep : StepEma<EMA> {
  float lr;
  float b1p, b2p;          // GACCUM_ADAM, GACCUM_LAMB: TF1's beta powers
  float bc2, bc1;          // GACCUM_ADAM: sqrt(1 - b2p) and 1 - b1p, the bias corrections of alpha_t (tile_rate)
  Divisor dv;              // apply launches: N, or the window weight W
  int ok;                  // 0: the device schedule refused the launch (sched_load)
};
static_assert(sizeof(LaunchStep<>) == 32, "the parts a kernel does not have take no space");

// Thread 0 of every CTA, before its CTA can reach a grid barrier or launch_commit -- so before any CTA of the launch can
// write what it reads, and every CTA finds the same step.  lr and the beta powers are the host's (Scalars), else the
// device schedule's; a loss-scaled launch takes the beta powers of the loss-scaling block, which advances them on
// applied windows only.  An accumulate launch (kAccumulate) reads the schedule alone; from_zero: it is a first accumulate.
template <int VARIANT, int MODE = kNoClip, bool EMA = false, typename KP>
__device__ __forceinline__ void launch_begin(const KP& prm, LaunchStep<EMA>& st, LossScaleState* ls = nullptr,
                                             const bool from_zero = false) {
  st.lr = prm.sc.lr;
  st.b1p = prm.sc.b1p;
  st.b2p = prm.sc.b2p;
  st.ok = 1;
  if (prm.sched.state) sched_load(prm.sched, prm.lrt, VARIANT != kAccumulate, from_zero, st);
  if constexpr (VARIANT != kAccumulate) {
    if constexpr (loss_scaled(MODE)) {
      ls_load(prm.ls.state, *ls);
      st.b1p = ls->beta1_power;
      st.b2p = ls->beta2_power;
    }
    if constexpr (EMA) ema_load(prm.ema, st.ema);
    st.dv = launch_divisor(prm);
    if constexpr (VARIANT == 1) {
      st.bc2 = __fsqrt_rn(__fsub_rn(1.0f, st.b2p));
      st.bc1 = __fsub_rn(1.0f, st.b1p);
    } else {
      st.bc2 = 1.0f;   // no alpha: tile_rate<0> does not read them
      st.bc1 = 1.0f;
    }
  }
}
// The one thread that commits a launch, once no CTA of it reads the state blocks any more: gaccum_stats (gn and s: the
// global norm and the clip scale, 0 and 1 without clipping), the loss-scaling state, the average (applied windows only),
// the window weight and the deferred reset's word (applied and skipped windows alike) and the schedule's next step.  The schedule advances the beta
// powers only where the launch took them from it: an optimizer that keeps them, on a launch that is not loss-scaled.
template <int VARIANT, int MODE = kNoClip, bool EMA = false, typename KP>
__device__ __forceinline__ void launch_commit(const KP& prm, const LaunchStep<EMA>& st, const LossScaleState* ls,
                                              const bool skip, const float gn, const float s) {
  constexpr bool apply = VARIANT != kAccumulate;
  prm.stats[0] = apply ? 1.f : 0.f; prm.stats[1] = st.lr; prm.stats[2] = gn; prm.stats[3] = s;
  if constexpr (loss_scaled(MODE)) ls_finish<keeps_beta_powers(VARIANT)>(prm.ls, *ls, skip, prm.sc.b1, prm.sc.b2);
  if constexpr (EMA) { if (!skip) ema_finish(prm.ema, st.ema); }
  if (apply && prm.ww.state) window_finish(prm.ww.state, st.dv.nf);
  if (apply && prm.dr.accum_zero) *prm.dr.accum_zero = 1u;   // deferred reset: the accumulators are +0 from here on
  if (prm.sched.state) sched_finish(prm.sched, keeps_beta_powers(VARIANT) && !loss_scaled(MODE), prm.sc.b1, prm.sc.b2);
}
// Thread 0 of every CTA of a one-tile-per-CTA launch, after its tile: true in the CTA that commits.  `counted` (the launch
// commits device state): the last CTA through, by a counter of finished CTAs -- every other CTA has read the state by
// then -- which it resets for the next launch.  Otherwise block 0, and nothing is counted.
__device__ __forceinline__ bool commits_launch(unsigned int* done, const bool counted) {
  if (!counted) return blockIdx.x == 0;
  __threadfence();
  if (atomicAdd(done, 1u) != gridDim.x - 1u) return false;
  *done = 0u;
  return true;
}

// Device schedule: every CTA checks the step before its tile, and the last one through commits the launch.  Without one
// the launch commits nothing but the stats, which no CTA reads: block 0 writes them before its tile, counting nothing.
// Deferred reset (FROM_ZERO only): every CTA reads the word before its tile.  All of them find the same value, since only
// this launch's last CTA through changes it: if it is 1, every CTA is counted and that last one clears it.
// gaccum_accum_materialize launches this kernel with no gradients and no schedule: a zero fill while the word is 1.
template <int CAP, bool FROM_ZERO, bool H = false>
__global__ void __launch_bounds__(kThreads)
accumulate_kernel(const __grid_constant__ KernelParams<CAP> prm) {
  __shared__ LaunchStep<> s_step;
  __shared__ unsigned int s_zero;
  const bool sched = prm.sched.state != nullptr;                     // launch-uniform
  const bool deferred = FROM_ZERO && prm.dr.accum_zero != nullptr;   // launch-uniform
  if (sched || deferred) {
    if (threadIdx.x == 0) {
      if (sched) launch_begin<kAccumulate>(prm, s_step, nullptr, FROM_ZERO);
      if (deferred) s_zero = __ldcg(prm.dr.accum_zero);
    }
    __syncthreads();
    if (sched && !s_step.ok) { sched_refuse(prm.sched); return; }
  }
  if (!sched && blockIdx.x == 0 && threadIdx.x == 0) {
    launch_begin<kAccumulate>(prm, s_step);
    launch_commit<kAccumulate>(prm, s_step, nullptr, false, 0.f, 1.f);
  }
  const bool zero = deferred && s_zero != 0u;
  if ((int)blockIdx.x < prm.num_tiles) accumulate_tile<FROM_ZERO, H>(prm.tiles[blockIdx.x], prm, zero);
  if ((sched || zero) && threadIdx.x == 0 && commits_launch(prm.done, true)) {
    if (sched) launch_commit<kAccumulate>(prm, s_step, nullptr, false, 0.f, 1.f);
    if (zero) *prm.dr.accum_zero = 0u;
  }
}

// gaccum_loss_scale_init: one thread writes the initial loss-scaling state (a kernel, so the call stays asynchronous and
// graph-capturable)
__global__ void loss_scale_init_kernel(LossScaleState* st, float scale, float b1, float b2) {
  LossScaleState s{};
  s.scale = scale;
  s.beta1_power = b1;
  s.beta2_power = b2;
  *st = s;
}

// gaccum_ema_init: n and d = 0, by one thread (asynchronous and graph-capturable, as loss_scale_init_kernel)
__global__ void ema_init_kernel(EmaState* st, long long num_updates) {
  EmaState s{};
  s.num_updates = num_updates;
  *st = s;
}

// ---------------------------------------------------------------------------------------------
// apply without clipping: one pass.  A tensor without a gradient applies its accumulator as it is.
// ---------------------------------------------------------------------------------------------
// H: p is the master slab (always 16-byte aligned); the model copy is stored after it.
// EMA: the average e (slab `ema`, always 16-byte aligned) is read with p and stored after it: e - (e - p) * c.
// dv: the launch's divisor (N, or the window weight W).
// lr, bc2, bc1: the step's learning rate and GACCUM_ADAM's bias-correction terms (LaunchStep).
// norms (launch-uniform, NormParams): the thread's fp32 partials of c^2 (c before any clip scale), p^2 (p before the
// update) and (p - p')^2 go into `np_`.
struct NormPart {
  float g = 0.f, w = 0.f, u = 0.f;
};
template <int VARIANT, bool H, int CAP, bool EMA = false>
__device__ __forceinline__ void update_tile(const TileDesc d, const KernelParams<CAP>& prm, const Divisor dv,
                                            const float lr, const float bc2, const float bc1, const bool norms,
                                            NormPart& np_, float* ema = nullptr, const float ema_c = 0.f) {
  const Grad<H> g(prm, d);
  const size_t soff = (size_t)d.soff32 * kSlabAlign;
  float* __restrict__ a = prm.accum + soff;
  float* __restrict__ m = prm.m + soff;
  float* __restrict__ v = prm.v + soff;
  float* __restrict__ p = update_ptr<H>(prm, d);
  float* __restrict__ e = EMA ? ema + soff : nullptr;
  uint16_t* q = nullptr;
  bool bf16 = false;
  if constexpr (H) { q = model_ptr(prm, d); bf16 = prm.half.bf16 != 0; }
  const bool decay = (d.tensor_flags >> 31) != 0;
  const bool deferred = prm.dr.accum_zero != nullptr;   // launch-uniform: a = +0 is not stored (DeferredResetParams)
  const Scalars& sc = prm.sc;
  const float rate = tile_rate<VARIANT>(lr, tensor_mult(prm.lrm, d), bc2, bc1);
  float4* a4 = reinterpret_cast<float4*>(a);
  float4* m4 = reinterpret_cast<float4*>(m);
  float4* v4 = reinterpret_cast<float4*>(v);
  float4* p4 = reinterpret_cast<float4*>(p);
  float4* e4 = reinterpret_cast<float4*>(e);
  float4 va[kUnroll], vg[kUnroll], vp[kUnroll], vm[kUnroll], vv[kUnroll], ve[kUnroll];
  // no gradient for this tile: a + 0 would turn -0 into +0 only; the add is skipped entirely (optimization.py:81)
  walk_tile(d.len, (H || aligned16(p)) && (g.g == nullptr || g.vec_ok()) ? d.len >> 2 : 0u, threadIdx.x,
            [&](int u, uint32_t i) {
              va[u] = __ldcs(a4 + i); vp[u] = __ldcs(p4 + i); vm[u] = __ldcs(m4 + i); vv[u] = __ldcs(v4 + i);
              if (g.g) vg[u] = g.vec(i);
              if constexpr (EMA) ve[u] = __ldcs(e4 + i);
            },
            [] {},
            [&](int u, uint32_t i) {
              if (g.g) va[u] = add_rn(va[u], vg[u]);
              float4 pb;
              if (norms) { np_.g = add_sq(np_.g, va[u], dv); np_.w = sq_acc(np_.w, vp[u]); pb = vp[u]; }
              update_vec<VARIANT>(va[u], false, 0.f, vp[u], vm[u], vv[u], decay, sc, rate, dv);
              if (norms) {
                np_.u = diff_sq_acc(diff_sq_acc(diff_sq_acc(diff_sq_acc(np_.u, pb.x, vp[u].x), pb.y, vp[u].y), pb.z, vp[u].z),
                                    pb.w, vp[u].w);
              }
              __stcs(p4 + i, vp[u]); __stcs(m4 + i, vm[u]); __stcs(v4 + i, vv[u]);
              if (!deferred) __stcs(a4 + i, make_float4(0.f, 0.f, 0.f, 0.f));   // optimization.py:86-87
              if constexpr (H) store_model4(q, i, vp[u], bf16);
              if constexpr (EMA) __stcs(e4 + i, ema_vec(ve[u], vp[u], ema_c));
            },
            [&](uint32_t i) {
              float ax = a[i], px = p[i], mx = m[i], vx = v[i];
              if (g.g) ax = __fadd_rn(ax, g.elem(i));
              const float pb = px;
              if (norms) { np_.g = add_sq(np_.g, ax, dv); np_.w = sq_acc(np_.w, px); }
              update_elem<VARIANT>(ax, false, 0.f, px, mx, vx, decay, sc, rate, dv);
              if (norms) np_.u = diff_sq_acc(np_.u, pb, px);
              p[i] = px; m[i] = mx; v[i] = vx;
              if (!deferred) a[i] = 0.f;
              if constexpr (H) q[i] = (uint16_t)f2h(px, bf16);
              if constexpr (EMA) e[i] = ema_elem(e[i], px, ema_c);
            });
}

// EMA, window weight and device schedule: every CTA reads the state before its tile (launch_begin); the CTA that
// finishes last commits the launch (commits_launch).
template <int VARIANT, int CAP, bool H = false, bool EMA = false>
__global__ void __launch_bounds__(kThreads)
apply_kernel(const __grid_constant__ KernelParams<CAP> prm) {
  __shared__ LaunchStep<EMA> s_step;
  const bool counted = EMA || prm.ww.state != nullptr || prm.sched.state != nullptr;   // launch-uniform
  if (threadIdx.x == 0) launch_begin<VARIANT, kNoClip, EMA>(prm, s_step);
  __syncthreads();
  if (!s_step.ok) { sched_refuse(prm.sched); return; }
  const Divisor dv = s_step.dv;
  const float lr = s_step.lr, bc2 = s_step.bc2, bc1 = s_step.bc1;
  const bool norms = prm.norms.out != nullptr;     // launch-uniform
  if ((int)blockIdx.x < prm.num_tiles) {
    const TileDesc d = prm.tiles[blockIdx.x];
    NormPart part;
    if constexpr (EMA) update_tile<VARIANT, H, CAP, true>(d, prm, dv, lr, bc2, bc1, norms, part, prm.ema.slab, s_step.ema.c);
    else update_tile<VARIANT, H>(d, prm, dv, lr, bc2, bc1, norms, part);
    if (norms) {
      const int warp = (int)threadIdx.x >> 5;
      norm_store(prm.norms, (int)blockIdx.x, 0, warp, part.g);
      norm_store(prm.norms, (int)blockIdx.x, 1, warp, part.w);
      norm_store(prm.norms, (int)blockIdx.x, 2, warp, part.u);
      norm_arrive_tile(prm.norms, d, (int)blockIdx.x);
    }
  }
  if (threadIdx.x == 0 && commits_launch(prm.done, counted)) launch_commit<VARIANT, kNoClip, EMA>(prm, s_step, nullptr, false, 0.f, 1.f);
}

// =============================================================================================
// apply with clipping: ONE cooperative launch, one CTA per SM =
//     3 consumer groups x 256 threads  +  3 producer warps (one per group)          (864 threads)
//
// NO consumer ever issues a bulk load: every input stream of both passes is moved by TMA
// (cp.async.bulk shared <- global, completing on an mbarrier by byte count) into a per-group ring in
// shared memory, fed by the group's producer warp.  Why:
//   * an LDG-fed pass can keep only as many bytes in flight as it has registers AND L1 lines to land them
//     in; L1 and shared memory split 256 KB per SM, so every KB of on-chip stash is paid for with bytes in
//     flight;
//   * TMA loads need neither registers nor L1: bytes in flight = ring size, descriptors and addresses are
//     computed by the producers ahead of the consumers, whose loop is wait -> LDS -> math -> store.
// NO tile is bound to an SM before it is fetched: with the memory system saturated some SMs get a larger share
// of it than others, so the producers draw tiles from global atomic ticket counters -- every SM stays busy until
// the pass is over.
//
// pass 1   the group's own tiles (the first kStashTiles of b, b + G, ... for group b of G) by position, then tickets
//          over all other tiles.  ring slot = [G tile | a tile] (16 KB, kP1Slots per group).  a' = a + G;
//          sum((a'/N)^2): thread fp32 per tile -> warp shuffle in fp64 (fixed order) -> EXACT accumulation of the
//          per-warp, per-tile sums in a 2176-bit fixed-point accumulator (integer atomics: associative, so the
//          total does not depend on which SM reduced which tile -- the norm is bit-identical from run to run
//          and across replicas although the schedule is dynamic).  a' of the group's own tiles is parked in the
//          group's shared-memory stash (the part of the SM's 227 KB the ring leaves free); every other a' goes
//          back in place tagged L2::evict_last.
// barrier  only the CONSUMERS rendezvous (named barrier + one atomic per CTA).  The producers do not: p, m, v do
//          not depend on the clip scale, so they start streaming the group's own stashed tiles into the
//          ring as soon as pass 1 is drained -- HBM stays busy while the CTAs wait for each other.
// pass 2   ring slot = [p | m | v | a'] (32 KB).  First the group's own stashed tiles, then tickets over
//          all other tiles, youngest first (a' still in L2): clip, AdamWeightDecay/Adam,
//          STG p, m, v, a = 0 (deferred reset: no a = 0, and a pool tile's a' lines are discarded from L2).
// Tiles that bulk copies cannot move (gradient / parameter pointer not 16-byte aligned, or shorter than one
// float4) go through the same full/empty protocol with nothing copied and are loaded by the consumers with
// scalar LDGs; producer and consumers evaluate the same predicates (bulk_vecs / bulk_vecs2).
// Per-launch counters (tickets, pool length, accumulator) exist twice; launch k uses set k & 1 and clears the
// other one, k being read off the monotonic barrier counter -- no host-side state, so launches replay in CUDA graphs.
// =============================================================================================
constexpr int kGroups = 3;                        // consumer groups per CTA
constexpr int kConsumerThreads = kThreads * kGroups;        // 768
constexpr int kClipThreads = kConsumerThreads + 32 * kGroups;   // + one producer warp per group = 864
constexpr int kP1Slots = 2;                       // pass-1 ring slots per group, 16 KB each
constexpr int kP1SlotVecs = 2 * (kTile / 4);      // float4 per pass-1 slot: G | a
constexpr int kP2SlotVecs = 4 * (kTile / 4);      // float4 per pass-2 slot: p | m | v | a'
constexpr int kRingVecs = kP1Slots * kP1SlotVecs; // per group
constexpr int kP2Slots = kRingVecs / kP2SlotVecs; // 2 x 16 KB = 32 KB -> 1 x 32 KB
constexpr int kRingBytes = kGroups * kRingVecs * 16;   // 96 KB
static_assert(kP2Slots >= 1, "ring must hold at least one [p|m|v|a'] slot");
// the stash: kStashTiles tiles of a' per group (8 KB each) in the shared memory the ring and the static arrays
// (~16 KB) leave free of the 227 KB a block may have on sm_90
constexpr int kStashTiles = 4;
static_assert(kStashTiles <= 32, "the producer loads the descriptors of a group's own tiles one per lane");
constexpr uint32_t kNoStash = 0xffffffffu;
constexpr int kStashVecs = kStashTiles * (kTile / 4);          // float4 per group
constexpr int kClipSmemBytes = kRingBytes + kGroups * kStashVecs * 16;   // dynamic shared memory of the kernel (192 KB)
static_assert(kClipSmemBytes + 20 * 1024 <= 227 * 1024, "ring + stash + static shared memory must fit one sm_90 block");
// The same shared memory laid out for either kind of launch.  An EMA launch moves a fifth stream, e, into its pass-2
// slot [p | m | v | a' | e] (40 KB): the ring grows to one such slot per group (pass 1 keeps its two 16 KB slots), and
// the stash shrinks to the tiles that then fit -- 3 per group instead of 4 -- so that no consumer issues a bulk load.
template <bool EMA>
struct ClipLayout {
  static constexpr int kP2SlotVecs = (EMA ? 5 : 4) * (kTile / 4);
  static constexpr int kRingVecs = kP1Slots * kP1SlotVecs > kP2SlotVecs ? kP1Slots * kP1SlotVecs : kP2SlotVecs;
  static constexpr int kP2Slots = kRingVecs / kP2SlotVecs;
  static constexpr int kRingBytes = kGroups * kRingVecs * 16;
  static constexpr int kStashTiles = (kClipSmemBytes - kRingBytes) / (kGroups * kTile * 4);
  static constexpr int kStashVecs = kStashTiles * (kTile / 4);
};
static_assert(ClipLayout<false>::kRingVecs == kRingVecs && ClipLayout<false>::kP2Slots == kP2Slots &&
              ClipLayout<false>::kStashTiles == kStashTiles, "the layout without an EMA is the one above");
static_assert(ClipLayout<true>::kP2Slots >= 1 && ClipLayout<true>::kStashTiles >= 1 &&
              ClipLayout<true>::kRingBytes + kGroups * ClipLayout<true>::kStashVecs * 16 <= kClipSmemBytes,
              "the EMA layout fits the same dynamic shared memory");
constexpr int kTicketBatch = 4;                   // pass-1 tickets a producer draws at once while plenty of tiles are left
// what the producer tells the consumers about the tile it put into a slot
struct __align__(16) SlotMeta {
  TileDesc d;          // len == 0: end of the pass
  uint32_t stash_slot; // pass 2: a' is parked in this stash slot of the group (kNoStash: it is in the slot's 4th quarter / in global memory)
  float rate;          // pass 2: the tile's lr_t (AdamWeightDecay) or alpha_t (Adam), tile_rate
  uint32_t tile;       // the tile's index in the table (per-tensor norms)
};
static_assert(sizeof(SlotMeta) == 32, "the rate and the tile index sit in what was padding: static shared memory is unchanged");
// exact accumulation of non-negative doubles: 68 bins of 32 payload bits in 64-bit containers cover the whole
// binary64 range (2^-1074 .. 2^1024); a container overflows only after 2^31 additions
constexpr int kAccBins = 68;
constexpr unsigned int kElemNonfinite = 4u;
struct LaunchCounters {
  unsigned long long p1_ticket, p2_ticket;
  unsigned int nonfinite, pad;                  // nonfinite: bit 0 = +inf seen, bit 1 = NaN seen (in the norm's sum),
                                                // bit 2 = a non-finite element of a' (loss-scaled launches only)
  unsigned long long bins[kAccBins];
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
               : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {}
}
// TMA bulk copy global -> shared, completion counted in bytes on `bar`
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar, uint64_t pol) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
               ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)), "l"(pol) : "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_gpu_u64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}

// ---------------------------------------------------------------------------------------------
// The stash: one CTA per SM by construction, so the shared memory the ring does not need holds a' of a
// group's first tiles from pass 1 to pass 2.  A stash slot keeps the tile in its natural float4 order,
// exactly like a ring slot, so thread t writes and later reads vectors t and t + kThreads of the tile:
// a thread only ever reads what it wrote itself (no barrier), and a warp touches 512 consecutive
// bytes per access (no bank conflicts).
// ---------------------------------------------------------------------------------------------

// Number of float4 vectors of this tile that pass 1 moves by bulk copy (0: scalar fallback).  The producer and
// the consumers MUST agree on this.
// A 16-bit G (H) moves in 16-byte granules of 8 elements, i.e. an even number of vectors: the G half of the slot holds
// nvec x 8 bytes of it.
template <bool H>
__device__ __forceinline__ uint32_t bulk_vecs(const TileDesc& d, const Grad<H>& g) {
  if constexpr (H) return g.g == nullptr ? (d.len >> 2) : aligned16(g.g) ? (d.len >> 3) << 1 : 0u;
  else return (g.g == nullptr || aligned16(g.g)) ? (d.len >> 2) : 0u;
}
// ... and that pass 2 moves by bulk copy (p: the parameters, or the master slab of a 16-bit model)
__device__ __forceinline__ uint32_t bulk_vecs2(const TileDesc& d, const float* p) {
  return aligned16(p) ? (d.len >> 2) : 0u;
}

// a' of a tile may be parked in the stash only if BOTH passes take the vector path for it and it is a full tile
template <bool H, int CAP>
__device__ __forceinline__ bool stash_ok(const TileDesc& d, const KernelParams<CAP>& prm) {
  bool ok = d.len == (uint32_t)kTile && aligned16(update_ptr<H>(prm, d));
  const Grad<H> g(prm, d);
  ok = ok && (g.g == nullptr || aligned16(g.g));
  return ok;
}

// one thread's view of a ring: slot index + how often the ring has wrapped
struct RingPos {
  int slot = 0;
  uint32_t use = 0;
  __device__ __forceinline__ void advance(int nslots) { if (++slot == nslots) { slot = 0; ++use; } }
};

// ---- exact accumulator ---------------------------------------------------------------------------------------
// add the non-negative double w to `bins` exactly; non-finite values only raise a flag.  `bins` is PRIVATE to the
// calling thread (one accumulator per warp, lane 0 owns it): plain read-modify-write, no atomics, no contention
__device__ __forceinline__ void acc_add(unsigned long long* bins, unsigned int& nonfinite, const double w) {
  const unsigned long long bits = (unsigned long long)__double_as_longlong(w);
  const unsigned int e = (unsigned int)(bits >> 52) & 0x7ffu;
  if (e == 0x7ffu) { nonfinite |= (bits & 0x000fffffffffffffull) ? 2u : 1u; return; }
  unsigned long long mant = bits & 0x000fffffffffffffull;
  if (e != 0) mant |= 1ull << 52;
  if (mant == 0) return;
  const unsigned int pos = e ? e - 1u : 0u;           // bit position of mant's LSB: value = mant * 2^(pos - 1074)
  const unsigned int q = pos >> 5, r = pos & 31u;
  const unsigned long long lo = mant << r;            // r <= 31, mant < 2^53: the 85-bit product is split by hand
  const unsigned long long hi = r ? (mant >> (64u - r)) : 0ull;
  bins[q] += lo & 0xffffffffull;
  bins[q + 1] += lo >> 32;
  bins[q + 2] += hi;
}
// the accumulated value as a double ROUNDED TO ODD: its leading 53 bits, the last one ORed with every bit below them
// (the rest of the three leading 32-bit digits and every lower digit).  53 >= 24 + 2, so the caller's (float) cast then
// rounds the exact sum to fp32 once -- to nearest, ties to even, inf from FLT_MAX + half an ulp -- where rounding to
// nearest twice can land one ulp off.  Deterministic (carries propagated low to high); executed by one thread.
__device__ __forceinline__ double acc_value(const unsigned long long* bins /* kAccBins */, const unsigned int nonfinite) {
  if (nonfinite & 2u) return __longlong_as_double(0x7ff8000000000000ll);
  if (nonfinite & 1u) return __longlong_as_double(0x7ff0000000000000ll);
  unsigned long long carry = 0;
  int top = -1;
  for (int i = 0; i < kAccBins; ++i) {
    const unsigned long long t = bins[i] + carry;
    carry = t >> 32;
    if (t & 0xffffffffull) top = i;
  }
  if (top < 0) return 0.0;
  carry = 0;
  unsigned int g0 = 0, g1 = 0, g2 = 0;                 // digits top-2, top-1, top
  bool sticky = false;                                 // a digit below top-2 is not zero
  for (int i = 0; i <= top; ++i) {
    const unsigned long long t = bins[i] + carry;
    const unsigned int digit = (unsigned int)(t & 0xffffffffull);
    carry = t >> 32;
    if (i < top - 2) sticky |= digit != 0u;
    if (i == top - 2) g0 = digit;
    if (i == top - 1) g1 = digit;
    if (i == top) g2 = digit;
  }
  // the 96 bits g2:g1:g0 shifted left until g2's leading one is bit 63 of `hi`; what falls off joins the sticky bit
  const int lz = __clz(g2);
  unsigned long long hi = (((unsigned long long)g2 << 32) | g1) << lz;
  if (lz) hi |= (unsigned long long)g0 >> (32 - lz);
  sticky |= (g0 << lz) != 0u;                          // 32-bit shift: the bits of g0 below hi
  const unsigned long long mant = (hi >> 11) | (unsigned long long)(sticky || (hi & 0x7ffull) != 0ull);
  return scalbn((double)mant, 32 * (top - 1) - lz - 1074 + 11);
}

// ---- pieces the cooperative apply kernels share (apply_clip_kernel, lamb_apply_kernel in gaccum_lamb.cuh) ----------
// block 0: the other counter set was used by the previous launch on this plan, which is complete: clear it for the next
// one (threads 64 .. 64 + sizeof(LaunchCounters) / 8)
__device__ __forceinline__ void clear_other_counters(LaunchCounters* counters, const uint32_t set) {
  if (blockIdx.x == 0 && threadIdx.x >= 64 && threadIdx.x < 64 + (int)(sizeof(LaunchCounters) / 8)) {
    reinterpret_cast<unsigned long long*>(counters + (set ^ 1u))[threadIdx.x - 64] = 0ull;
  }
}
// grid barrier, executed by ONE thread per CTA: one atomic on a monotonic counter (every launch on a plan uses the same
// grid, so the counter advances by gridDim.x per barrier); cooperative launch guarantees that all CTAs are co-resident
__device__ __forceinline__ void grid_barrier(unsigned long long* barrier) {
  __threadfence();
  const unsigned long long old = atomicAdd(barrier, 1ull);
  const unsigned long long target = (old / gridDim.x + 1ull) * gridDim.x;
  while (ld_acquire_gpu_u64(barrier) < target) { __nanosleep(20); }
}
// thread 0 after the barrier, from the launch-wide counters (`bins`: their accumulator, copied where the thread reads
// it): the clip scale s and the global norm gn (1 and 0 without clipping) and, loss-scaled, whether the window is
// skipped -- an element of a' or, with clipping, gn is not finite.  Every CTA computes the same values.
template <int MODE>
__device__ __forceinline__ void window_decision(const LaunchCounters* ctr, const unsigned long long* bins, const float clip,
                                                float& s, float& gn, int& skip) {
  if constexpr (MODE == kLsNoClip) {
    s = 1.f;                                              // no clipping: stats as the un-clipped apply writes them
    gn = 0.f;
    skip = (__ldcg(&ctr->nonfinite) & kElemNonfinite) != 0;
  } else {
    const unsigned int nonfinite = __ldcg(&ctr->nonfinite);
    const double tot = acc_value(bins, nonfinite);
    const float g_norm = __fsqrt_rn((float)tot);          // tf.linalg.global_norm
    s = clip_scale(g_norm, clip);
    gn = g_norm;
    if constexpr (loss_scaled(MODE)) skip = (nonfinite & kElemNonfinite) != 0 || !(fabsf(g_norm) <= 3.402823466e38f);
  }
}

// ---- pass 1, consumer side: one tile out of slot [G | a]; returns this THREAD's partial of sum((a'/N)^2) ----
// A tile the producer did not copy (nvec == 0), and the < 4 tail elements of any tile, travel through global memory.
// Loss-scaled (kLsClip, kLsNoClip): the partial is of sum(((a'/N)(1/S))^2) (none without clipping), and `bad` is set
// when an element of a' is not finite.
// norms (kLsNoClip only; launch-uniform): the partial of sum(((a'/N)(1/S))^2) is formed as kLsClip forms it.
template <int MODE, bool H, int CAP>
__device__ __forceinline__ float norm_tile(const TileDesc& d, const KernelParams<CAP>& prm, const float4* slot, uint64_t* empty,
                                           float4* const stash, const uint64_t pol, const float inv_s, bool& bad,
                                           const Divisor& dv, const bool norms) {
  const Grad<H> g(prm, d);
  float* __restrict__ a = prm.accum + (size_t)d.soff32 * kSlabAlign;
  float4* a4 = reinterpret_cast<float4*>(a);
  float acc = 0.f;
  float4 x[kUnroll], gg[kUnroll];
  walk_tile(d.len, bulk_vecs(d, g), threadIdx.x & (kThreads - 1),
            [&](int u, uint32_t i) { x[u] = slot[kTile / 4 + i]; if (g.g) gg[u] = g.slot(slot, i); },
            [&] { __syncwarp(); if ((threadIdx.x & 31) == 0) mbar_arrive(empty); },   // this warp is done with the slot
            [&](int u, uint32_t i) {
              if (g.g) {
                x[u] = add_rn(x[u], gg[u]);
                if (stash == nullptr) st_policy(a4 + i, x[u], pol);
              }
              if (stash != nullptr) stash[i] = x[u];
              if constexpr (!loss_scaled(MODE)) acc = add_sq(acc, x[u], dv);
              else if (MODE == kLsNoClip && norms) acc = ls_pass1<kLsClip>(acc, x[u], inv_s, bad, dv);
              else acc = ls_pass1<MODE>(acc, x[u], inv_s, bad, dv);
            },
            [&](uint32_t i) {
              float xs = a[i];
              if (g.g) { xs = __fadd_rn(xs, g.elem(i)); a[i] = xs; }
              if constexpr (!loss_scaled(MODE)) acc = add_sq(acc, xs, dv);
              else if (MODE == kLsNoClip && norms) acc = ls_pass1<kLsClip>(acc, xs, inv_s, bad, dv);
              else acc = ls_pass1<MODE>(acc, xs, inv_s, bad, dv);
            });
  return acc;
}

// ---- pass 2, consumer side: one tile out of slot [p | m | v | a']; a' from the slot or from the stash ----
// The caller has waited on the slot's `full` barrier (it had to, to learn which tile this is).
// `rate` is the tile's lr_t / alpha_t (SlotMeta::rate; loss-scaled Adam: from the device's beta powers).
// Loss-scaled: a skipped window (`skip`) stores a = 0 and nothing else.  H: p is the master slab, and the model copy is
// stored after it (not on a skipped window).
// Deferred reset (DeferredResetParams): a = 0 is not stored, and a pool tile's a' lines are discarded from L2.
// EMA: the slot is [p | m | v | a' | e], and e - (e - p) * c is stored after p (not on a skipped window).
// norms (launch-uniform): the slot is kept for norm_tile2 instead of being released after the loads, and the tile's
// elements in it are made those norm_tile2 reads -- p before the update in the slot's p quarter (where the vector path
// already has it), the stored p' in its m quarter (consumed by then), element i at float i -- so that no value is kept
// alive across the update, whose registers are the kernel's limit.
template <int VARIANT, int MODE, bool H, int CAP, bool EMA = false>
__device__ __forceinline__ void update_tile2(const TileDesc& d, const KernelParams<CAP>& prm, const float s, float4* slot,
                                             uint64_t* empty, const float4* const stash, const float rate, const float inv_s,
                                             const bool skip, const Divisor& dv, const bool norms,
                                             float* ema = nullptr, const float ema_c = 0.f) {
  const Scalars& sc = prm.sc;
  const size_t soff = (size_t)d.soff32 * kSlabAlign;
  float* __restrict__ a = prm.accum + soff;
  float* __restrict__ m = prm.m + soff;
  float* __restrict__ v = prm.v + soff;
  float* __restrict__ p = update_ptr<H>(prm, d);
  float* __restrict__ e = EMA ? ema + soff : nullptr;
  uint16_t* q = nullptr;
  bool bf16 = false;
  if constexpr (H) { q = model_ptr(prm, d); bf16 = prm.half.bf16 != 0; }
  const bool decay = (d.tensor_flags >> 31) != 0;
  const bool write = !loss_scaled(MODE) || !skip;
  const bool deferred = prm.dr.accum_zero != nullptr;   // launch-uniform: a = +0 is not stored (DeferredResetParams)
  float4* a4 = reinterpret_cast<float4*>(a);
  float4* m4 = reinterpret_cast<float4*>(m);
  float4* v4 = reinterpret_cast<float4*>(v);
  float4* p4 = reinterpret_cast<float4*>(p);
  float4* e4 = reinterpret_cast<float4*>(e);
  float4 va[kUnroll], vp[kUnroll], vm[kUnroll], vv[kUnroll], ve[kUnroll];
  const uint32_t nvec = bulk_vecs2(d, p);
  if (deferred && stash == nullptr) {
    // a' of a pool tile has landed in the slot: its whole lines in global memory are dead (a tail line still holds
    // elements the scalar path reads below), and dropping them saves the write-back of those still in L2
    const uint32_t line = threadIdx.x & (kThreads - 1);
    if (line < nvec / 8u) discard_line(a + 32u * line);
  }
  walk_tile(d.len, nvec, threadIdx.x & (kThreads - 1),
            [&](int u, uint32_t i) {
              vp[u] = slot[i]; vm[u] = slot[kTile / 4 + i]; vv[u] = slot[2 * (kTile / 4) + i];
              va[u] = stash != nullptr ? stash[i] : slot[3 * (kTile / 4) + i];
              if constexpr (EMA) ve[u] = slot[4 * (kTile / 4) + i];
            },
            [&] { if (!norms) { __syncwarp(); if ((threadIdx.x & 31) == 0) mbar_arrive(empty); } },
            [&](int u, uint32_t i) {
              if (write) {
                adam_vec<VARIANT, MODE>(va[u], s, inv_s, vp[u], vm[u], vv[u], decay, sc, rate, dv);
                __stcs(p4 + i, vp[u]); __stcs(m4 + i, vm[u]); __stcs(v4 + i, vv[u]);
                if constexpr (H) store_model4(q, i, vp[u], bf16);
                if constexpr (EMA) __stcs(e4 + i, ema_vec(ve[u], vp[u], ema_c));
                if (norms) slot[kTile / 4 + i] = vp[u];
              }
              if (!deferred) __stcs(a4 + i, make_float4(0.f, 0.f, 0.f, 0.f));   // optimization.py:86-87
            },
            [&](uint32_t i) {
              float* const sf = reinterpret_cast<float*>(slot);
              if (write) {
                float px = p[i], mx = m[i], vx = v[i];
                if (norms) sf[i] = px;
                adam_elem<VARIANT>(mode_c<MODE>(a[i], s, inv_s, dv), px, mx, vx, decay, sc, rate);
                p[i] = px; m[i] = mx; v[i] = vx;
                if (norms) sf[kTile + i] = px;
                if constexpr (H) q[i] = (uint16_t)f2h(px, bf16);
                if constexpr (EMA) e[i] = ema_elem(e[i], px, ema_c);
              } else if (norms) {
                sf[i] = p[i];
              }
              if (!deferred) a[i] = 0.f;
            });
}
// norms, after update_tile2: the tile's partials of p^2 (p before the update) and, unless the window is skipped,
// (p - p')^2 from what update_tile2 left in the slot.  Each thread reads exactly the elements it wrote (walk_tile's
// assignment, nvec as update_tile2 took it), so no barrier is needed.  Then the slot goes back to the producer: it was
// written through the generic proxy and the producer's next bulk copy into it is an async-proxy write, hence the proxy
// fence before the release.
__device__ __forceinline__ void norm_tile2(const TileDesc& d, const uint32_t nvec, const float4* slot, uint64_t* empty,
                                           const bool skip, float& nw, float& nu) {
  const uint32_t tid = threadIdx.x & (kThreads - 1);
#pragma unroll
  for (int u = 0; u < kUnroll; ++u) {
    const uint32_t i = u * kThreads + tid;
    if (i < nvec) {
      const float4 pb = slot[i];
      nw = sq_acc(nw, pb);
      if (!skip) {
        const float4 pn = slot[kTile / 4 + i];
        nu = diff_sq_acc(diff_sq_acc(diff_sq_acc(diff_sq_acc(nu, pb.x, pn.x), pb.y, pn.y), pb.z, pn.z), pb.w, pn.w);
      }
    }
  }
  const float* const sf = reinterpret_cast<const float*>(slot);
  for (uint32_t i = (nvec << 2) + tid; i < d.len; i += kThreads) {
    const float pb = sf[i];
    nw = sq_acc(nw, pb);
    if (!skip) nu = diff_sq_acc(nu, pb, sf[kTile + i]);
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncwarp();
  if ((threadIdx.x & 31) == 0) mbar_arrive(empty);
}

// Dynamic shared memory of apply_clip_kernel (kClipSmemBytes): 3 groups x kRingVecs float4 of ring, then
// 3 groups x kStashVecs float4 of stash.
// Registers: 864 threads in one CTA cap the kernel at 72 per thread.  ptxas -v (CUDA 12.9): only the fp32 AdamWeightDecay
// kClip instantiations without an EMA fit without spilling (the 16-bit ones store 8 bytes per thread since the deferred
// reset).  Every other one spills: AdamWeightDecay 4-24 bytes of stores per thread loss-scaled, 44-68 with an EMA; plain
// Adam (VARIANT 1) 8-44 without an EMA, 52-80 with one.  What that costs has not been measured.
//
// Device state (loss scaling, EMA, window weight, device schedule): thread 0 of every CTA reads it during set-up
// (launch_begin), before its CTA arrives at the grid barrier; block 0's thread 0 commits the launch at the very end
// (launch_commit) -- after the barrier, so no CTA can see a new value in this launch.
//
// Loss scaling (kLsClip, kLsNoClip; gaccum_plan_set_loss_scale): pass 1 ORs kElemNonfinite into the launch's counters
// when an element of a' is not finite.  After the barrier every CTA takes the same decision from the same launch-wide
// flags: skip iff an element was non-finite or, with clipping, gn is.  A skipped window stores a = 0 and leaves p, m and
// v alone.
//
// 16-bit models (H): pass 1 moves the 16-bit G tile into the G half of the [G | a] slot (bulk_vecs), pass 2 moves the
// master weights, and every store of p is followed by the model copy.  Ring and stash are the same.
//
// EMA: ClipLayout<true> -- pass 2's producer moves e by bulk copy as the fifth stream of the slot.
template <int VARIANT, int CAP, int MODE, bool H = false, bool EMA = false>
__global__ void __launch_bounds__(kClipThreads, 1)
apply_clip_kernel(const __grid_constant__ KernelParams<CAP> prm) {
  using L = ClipLayout<EMA>;
  constexpr int kRingVecs = L::kRingVecs, kP2SlotVecs = L::kP2SlotVecs, kP2Slots = L::kP2Slots, kRingBytes = L::kRingBytes;
  constexpr int kStashTiles = L::kStashTiles, kStashVecs = L::kStashVecs;
  const EmaParams* const ema = &prm.ema;   // read through a pointer: without it nvcc adds instructions to one EMA instantiation
  extern __shared__ __align__(128) unsigned char smem_dyn[];
  __shared__ unsigned long long s_bins[kConsumerThreads / 32][kAccBins];   // one exact accumulator per consumer warp (13 KB)
  __shared__ unsigned int s_nonfinite;
  __shared__ float s_bcast[2];
  __shared__ LaunchStep<EMA> s_step;
  __shared__ LossScaleState s_ls;        // loss-scaled: the state as this launch found it
  __shared__ int s_skip;
  __shared__ uint32_t s_set;
  __shared__ __align__(8) uint64_t s_full1[kGroups][kP1Slots], s_empty1[kGroups][kP1Slots];
  __shared__ __align__(8) uint64_t s_full2[kGroups][kP2Slots], s_empty2[kGroups][kP2Slots];
  __shared__ __align__(8) uint64_t s_go[kGroups];
  __shared__ SlotMeta s_meta1[kGroups][kP1Slots], s_meta2[kGroups][kP2Slots];

  const int warp = (int)threadIdx.x >> 5;
  const bool is_producer = warp >= kConsumerThreads / 32;
  const int grp = is_producer ? warp - kConsumerThreads / 32 : (int)threadIdx.x / kThreads;   // group served / group id
  const int nt = prm.num_tiles, G = (int)gridDim.x * kGroups;
  const int b = (int)blockIdx.x * kGroups + grp;                   // virtual block id
  const int C = b < nt ? (nt - 1 - b) / G + 1 : 0;                 // tiles b, b + G, ... below nt
  const int n_st = min(kStashTiles, C);                            // own tiles: a' parked in the stash
  const int pool_lo = min(nt, kStashTiles * G);                    // tiles [pool_lo, nt): a' goes back to global memory
  float4* const ring = reinterpret_cast<float4*>(smem_dyn) + (size_t)grp * kRingVecs;
  float4* const stash = reinterpret_cast<float4*>(smem_dyn + kRingBytes) + (size_t)grp * kStashVecs;
  const uint64_t pol_last = policy_evict_last();

#ifdef GACCUM_EXPERIMENTS
  auto stamp = [&](int which) {
    if (prm.debug && threadIdx.x == 0) {
      unsigned long long t;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
      prm.debug[blockIdx.x * 16 + which] = t;
    }
  };
#else
  auto stamp = [](int) {};
#endif
  stamp(0);

  // ---- set-up: which counter set this launch uses, mbarriers, accumulator -----------------------------------
  const bool norms = prm.norms.out != nullptr;   // launch-uniform: one more grid barrier at the end of the launch
  if (threadIdx.x == 0) {
    // every CTA that has not yet arrived at this launch's first barrier reads a value in [k*B*grid, (k*B+1)*grid), B the
    // launch's barriers
    const unsigned long long k = ld_acquire_gpu_u64(prm.barrier) / ((unsigned long long)gridDim.x * (norms ? 2ull : 1ull));
    s_set = (uint32_t)(k & 1ull);
    s_nonfinite = 0;
#pragma unroll
    for (int g = 0; g < kGroups; ++g) {
      for (int sl = 0; sl < kP1Slots; ++sl) { mbar_init(&s_full1[g][sl], 1); mbar_init(&s_empty1[g][sl], kThreads / 32); }
      for (int sl = 0; sl < kP2Slots; ++sl) { mbar_init(&s_full2[g][sl], 1); mbar_init(&s_empty2[g][sl], kThreads / 32); }
      mbar_init(&s_go[g], 1);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    launch_begin<VARIANT, MODE, EMA>(prm, s_step, &s_ls);
  }
  for (int i = threadIdx.x; i < (kConsumerThreads / 32) * kAccBins; i += kClipThreads) (&s_bins[0][0])[i] = 0ull;
  __syncthreads();
  // device schedule: every CTA read the same step, so all of them leave here or none does (before any barrier)
  if (!s_step.ok) { sched_refuse(prm.sched); return; }
  LaunchCounters* const ctr = prm.counters + s_set;
  clear_other_counters(prm.counters, s_set);

  if (is_producer) {
    // =========================== producer warp of group `grp` ===========================
    const int lane = (int)threadIdx.x & 31;
    const uint64_t pol_first = policy_evict_first();
#ifdef GACCUM_EXPERIMENTS
    long long dbg_empty = 0;
    const long long dbg_p0 = clock64();
#endif
    // ---- pass 1.  First the group's OWN tiles b + j*G, j < kStashTiles: their a' is parked in this SM's stash, so
    //      they are bound to it in both passes.  Then the rest of the model, tiles [pool_lo, nt), as the global ticket
    //      counter hands them out -- kTicketBatch tickets at a time while plenty are left (one atomic per lane, the
    //      descriptor loads of a batch overlap), single tickets near the end so that no SM is left holding a batch ----
    {
      RingPos rp;
      auto issue = [&](const TileDesc& dl, const int tile) {               // lane 0 only
        const Grad<H> g(prm, dl);
        const uint32_t nvec = bulk_vecs(dl, g);
        uint64_t* full = &s_full1[grp][rp.slot];
#ifdef GACCUM_EXPERIMENTS
        const long long t_e0 = clock64();
#endif
        mbar_wait(&s_empty1[grp][rp.slot], rp.use & 1u);             // the consumers have released the slot
#ifdef GACCUM_EXPERIMENTS
        dbg_empty += clock64() - t_e0;
#endif
        SlotMeta* meta = &s_meta1[grp][rp.slot];
        meta->d = dl;
        meta->tile = (uint32_t)tile;
        if (nvec > 0) {
          float4* dst = ring + (size_t)rp.slot * kP1SlotVecs;
          if constexpr (H) {
            mbar_arrive_expect_tx(full, nvec * 16u + (g.g ? nvec * 8u : 0u));
            if (g.g) bulk_g2s(dst, g.g, nvec * 8u, full, pol_first);
          } else {
            mbar_arrive_expect_tx(full, nvec * 16u * (g.g ? 2u : 1u));
            if (g.g) bulk_g2s(dst, g.g, nvec * 16u, full, pol_first);
          }
          bulk_g2s(dst + kTile / 4, prm.accum + (size_t)dl.soff32 * kSlabAlign, nvec * 16u, full, pol_first);
        } else {
          mbar_arrive(full);                                                 // nothing to copy: complete the phase
        }
      };
      auto shuffled = [&](const TileDesc& d, int l) {
        TileDesc dl;
        dl.tensor_flags = __shfl_sync(0xffffffffu, d.tensor_flags, l);
        dl.len = __shfl_sync(0xffffffffu, d.len, l);
        dl.toff = __shfl_sync(0xffffffffu, d.toff, l);
        dl.soff32 = __shfl_sync(0xffffffffu, d.soff32, l);
        return dl;
      };
      {
        TileDesc d{};
        if (lane < n_st) d = prm.tiles[b + lane * G];                        // own tiles' descriptors, one per lane
        for (int l = 0; l < n_st; ++l) {
          const TileDesc dl = shuffled(d, l);
          if (lane == 0) issue(dl, b + l * G);
          rp.advance(kP1Slots);
        }
      }
      bool done = false;
      long long last = pool_lo;
      while (!done) {
        const long long left = (long long)nt - last;
        const int batch = left > 8ll * G ? kTicketBatch : (left > 2ll * G ? 2 : 1);
        long long tile = nt;
        TileDesc d{};
        if (lane < batch) {
          tile = (long long)pool_lo + (long long)atomicAdd(&ctr->p1_ticket, 1ull);
          if (tile < nt) d = prm.tiles[tile];
        }
        for (int l = 0; l < batch; ++l) {
          const long long tl = __shfl_sync(0xffffffffu, tile, l);
          if (tl >= nt) { done = true; continue; }       // lanes get their tickets in no particular order: a valid one may follow
          last = tl;
          const TileDesc dl = shuffled(d, l);
          if (lane == 0) issue(dl, (int)tl);
          rp.advance(kP1Slots);
        }
      }
      if (lane == 0) {
        // end marker, then drain: pass 2's slots overlay pass 1's, so every slot must have been released for the last time
        mbar_wait(&s_empty1[grp][rp.slot], rp.use & 1u);
        s_meta1[grp][rp.slot].d.len = 0;
        mbar_arrive(&s_full1[grp][rp.slot]);
        for (int sl = 0; sl < kP1Slots; ++sl) {
          if (sl == rp.slot) continue;
          const uint32_t n = rp.use + (sl < rp.slot ? 1u : 0u);              // times slot sl was armed
          if (n > 0) mbar_wait(&s_empty1[grp][sl], n & 1u);
        }
      }
      __syncwarp();
    }
#ifdef GACCUM_EXPERIMENTS
    if (prm.debug && lane == 0) {
      prm.debug[blockIdx.x * 16 + 7 + grp] = (unsigned long long)dbg_empty;               // cycles the producer waited for a free slot
      prm.debug[blockIdx.x * 16 + 13 + grp] = (unsigned long long)(clock64() - dbg_p0);   // cycles until pass 1 was issued and drained
    }
#endif
    // ---- pass 2.  First the group's own stashed tiles (their a' cannot move; their p, m, v do not depend on
    //      the clip scale, so these copies start BEFORE the grid barrier and HBM stays busy while the CTAs wait for
    //      each other).  Then tickets over the pool of L2-resident tiles, youngest first.  Pool tiles carry their a'
    //      in the slot's 4th quarter; they may only be fetched once every CTA has passed the barrier. ----
    if (lane == 0) {
      RingPos rp;
      int jb = 0;
      bool past_barrier = false;
      const float lr = s_step.lr, bc2 = s_step.bc2, bc1 = s_step.bc1;
      const unsigned long long pool_n = (unsigned long long)max(0, nt - pool_lo);
      while (true) {
        int tile;
        uint32_t stash_slot = kNoStash;
        if (jb < n_st) {
          tile = b + jb * G;
          stash_slot = (uint32_t)jb;
          ++jb;
        } else {
          if (!past_barrier) {
            mbar_wait(&s_go[grp], 0);                                           // the consumers are through the grid barrier
            asm volatile("fence.proxy.async;" ::: "memory");                    // generic-proxy a' stores -> our bulk reads
            past_barrier = true;
          }
          const unsigned long long tk = atomicAdd(&ctr->p2_ticket, 1ull);
          if (tk >= pool_n) break;
          tile = nt - 1 - (int)tk;                                              // youngest a' lines first
        }
        const TileDesc d = prm.tiles[tile];
        const float* p = update_ptr<H>(prm, d);
        const uint32_t nvec = bulk_vecs2(d, p);
        const bool in_stash = stash_slot != kNoStash && stash_ok<H>(d, prm);
        if (!in_stash && !past_barrier) {                                        // an own tile whose a' had to go to global memory
          mbar_wait(&s_go[grp], 0);
          asm volatile("fence.proxy.async;" ::: "memory");
          past_barrier = true;
        }
        uint64_t* full = &s_full2[grp][rp.slot];
        mbar_wait(&s_empty2[grp][rp.slot], rp.use & 1u);
        SlotMeta* meta = &s_meta2[grp][rp.slot];
        meta->d = d;
        meta->tile = (uint32_t)tile;
        meta->stash_slot = in_stash ? stash_slot : kNoStash;
        meta->rate = tile_rate<VARIANT>(lr, tensor_mult(prm.lrm, d), bc2, bc1);
        if (nvec > 0) {
          const size_t soff = (size_t)d.soff32 * kSlabAlign;
          float4* dst = ring + (size_t)rp.slot * kP2SlotVecs;
          if constexpr (EMA) mbar_arrive_expect_tx(full, nvec * 16u * (in_stash ? 4u : 5u));
          else mbar_arrive_expect_tx(full, nvec * 16u * (in_stash ? 3u : 4u));
          bulk_g2s(dst, p, nvec * 16u, full, pol_first);
          bulk_g2s(dst + kTile / 4, prm.m + soff, nvec * 16u, full, pol_first);
          bulk_g2s(dst + 2 * (kTile / 4), prm.v + soff, nvec * 16u, full, pol_first);
          if (!in_stash) bulk_g2s(dst + 3 * (kTile / 4), prm.accum + soff, nvec * 16u, full, pol_first);
          if constexpr (EMA) bulk_g2s(dst + 4 * (kTile / 4), ema->slab + soff, nvec * 16u, full, pol_first);
        } else {
          mbar_arrive(full);
        }
        rp.advance(kP2Slots);
      }
      mbar_wait(&s_empty2[grp][rp.slot], rp.use & 1u);                   // end marker
      s_meta2[grp][rp.slot].d.len = 0;
      mbar_arrive(&s_full2[grp][rp.slot]);
    }
    __syncwarp();
  } else {
    // =========================== consumer group ===========================
#ifdef GACCUM_EXPERIMENTS
    long long dbg_wait = 0;
    const long long dbg_t0 = clock64();
#endif
    const bool leader = (threadIdx.x & (kThreads - 1)) == 0;
    // every slot starts out empty: the consumers say so (phase 0 of each `empty` barrier), so that the producer's very
    // first wait is an ordinary wait on a phase that completes -- use u of a slot waits for phase u
    if ((threadIdx.x & 31) == 0) {
      for (int sl = 0; sl < kP1Slots; ++sl) mbar_arrive(&s_empty1[grp][sl]);
      for (int sl = 0; sl < kP2Slots; ++sl) mbar_arrive(&s_empty2[grp][sl]);
    }
    // ---- pass 1: whatever tiles the producer hands over, until its end marker ----
    unsigned int my_nonfinite = 0;
    float inv_s = 1.0f;
    if constexpr (loss_scaled(MODE)) inv_s = __fdiv_rn(1.0f, s_ls.scale);   // exact: S is a power of two
    {
      RingPos rp;
      int n_seen = 0;
      while (true) {
#ifdef GACCUM_EXPERIMENTS
        const long long t_w0 = clock64();
#endif
        mbar_wait(&s_full1[grp][rp.slot], rp.use & 1u);
#ifdef GACCUM_EXPERIMENTS
        dbg_wait += clock64() - t_w0;
#endif
        const SlotMeta meta = s_meta1[grp][rp.slot];
        if (meta.d.len == 0) break;
        // the stash takes the group's own tiles j < kStashTiles (the first ones it is handed) when they are FULL,
        // vector-path tiles (the same predicate the producer evaluates in pass 2)
        const bool own = n_seen < n_st;
        const bool park = own && stash_ok<H>(meta.d, prm);
        float4* const st = park ? stash + (size_t)n_seen * (kTile / 4) : nullptr;
        bool bad = false;
        const float part = norm_tile<MODE, H>(meta.d, prm, ring + (size_t)rp.slot * kP1SlotVecs, &s_empty1[grp][rp.slot], st,
                                                pol_last, inv_s, bad, s_step.dv, norms);
        if constexpr (loss_scaled(MODE)) { if (bad) my_nonfinite |= kElemNonfinite; }
        if (MODE != kLsNoClip || norms) {
          // warp total in fp64, fixed butterfly order; lane 0 adds it EXACTLY into its warp's accumulator and, with
          // norms, stores it as the tile's gradient partial of this warp
          double w = (double)part;
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) w += __shfl_xor_sync(0xffffffffu, w, o);
          if ((threadIdx.x & 31) == 0) {
            if constexpr (MODE != kLsNoClip) acc_add(s_bins[warp], my_nonfinite, w);
            if (norms) {
              prm.norms.tile_part[((size_t)meta.tile * kNormCols) * kNormWarps + (warp & (kNormWarps - 1))] = w;
            }
          }
        }
        ++n_seen;
        rp.advance(kP1Slots);
      }
    }
#ifdef GACCUM_EXPERIMENTS
    if (prm.debug && leader) {
      prm.debug[blockIdx.x * 16 + 4 + grp] = (unsigned long long)dbg_wait;                 // cycles waiting for G | a
      prm.debug[blockIdx.x * 16 + 10 + grp] = (unsigned long long)(clock64() - dbg_t0);   // cycles of the group's pass 1
    }
#endif
    named_bar_sync(1, kConsumerThreads);                     // every consumer thread of this CTA is through pass 1
    // flush this CTA's accumulators into the launch's global one (integer adds: order does not matter)
    if (my_nonfinite) atomicOr(&s_nonfinite, my_nonfinite);
    if (threadIdx.x < kAccBins) {
      unsigned long long v = 0;
      for (int w = 0; w < kConsumerThreads / 32; ++w) v += s_bins[w][threadIdx.x];
      if (v) atomicAdd(&ctr->bins[threadIdx.x], v);
    }
    named_bar_sync(1, kConsumerThreads);
    if (threadIdx.x == 0 && s_nonfinite) atomicOr(&ctr->nonfinite, s_nonfinite);
    stamp(1);
    // ---- grid barrier of the consumers (grid_barrier: one atomic per CTA on the plan's monotonic counter) ----
    if (threadIdx.x == 0) grid_barrier(prm.barrier);
    named_bar_sync(1, kConsumerThreads);
    if (leader) mbar_arrive(&s_go[grp]);                     // this group's producer may now fetch pool tiles
    stamp(2);
    // ---- every CTA evaluates the same exact sum the same way: bit-identical gn and clip scale everywhere ----
    if constexpr (MODE != kLsNoClip) {
      if (threadIdx.x < kAccBins) s_bins[0][threadIdx.x] = __ldcg(&ctr->bins[threadIdx.x]);
      named_bar_sync(1, kConsumerThreads);
    }
    if (threadIdx.x == 0) window_decision<MODE>(ctr, s_bins[0], prm.sc.clip, s_bcast[0], s_bcast[1], s_skip);
    named_bar_sync(1, kConsumerThreads);
    const float s = s_bcast[0];
    bool skip = false;
    if constexpr (loss_scaled(MODE)) skip = s_skip != 0;
    // ---- pass 2: whatever tiles the producer hands over, until its end marker ----
    {
      RingPos rp;
      while (true) {
        mbar_wait(&s_full2[grp][rp.slot], rp.use & 1u);
        const SlotMeta meta = s_meta2[grp][rp.slot];
        if (meta.d.len == 0) break;
        const float4* const st = meta.stash_slot != kNoStash ? stash + (size_t)meta.stash_slot * (kTile / 4) : nullptr;
        if constexpr (EMA) {
          update_tile2<VARIANT, MODE, H, CAP, true>(meta.d, prm, s, ring + (size_t)rp.slot * kP2SlotVecs, &s_empty2[grp][rp.slot],
                                                    st, meta.rate, inv_s, skip, s_step.dv, norms, ema->slab, s_step.ema.c);
        } else {
          update_tile2<VARIANT, MODE, H>(meta.d, prm, s, ring + (size_t)rp.slot * kP2SlotVecs, &s_empty2[grp][rp.slot], st, meta.rate,
                                      inv_s, skip, s_step.dv, norms);
        }
        if (norms) {
          float nw = 0.f, nu = 0.f;
          norm_tile2(meta.d, bulk_vecs2(meta.d, update_ptr<H>(prm, meta.d)), ring + (size_t)rp.slot * kP2SlotVecs,
                     &s_empty2[grp][rp.slot], loss_scaled(MODE) && skip, nw, nu);
          norm_store(prm.norms, (int)meta.tile, 1, warp & (kNormWarps - 1), nw);
          norm_store(prm.norms, (int)meta.tile, 2, warp & (kNormWarps - 1), nu);
        }
        rp.advance(kP2Slots);
      }
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) launch_commit<VARIANT, MODE, EMA>(prm, s_step, &s_ls, skip, s_bcast[1], s);
    if (norms) {
      // every tile's partials are stored once all consumers are through pass 2: a second grid barrier, then every
      // consumer warp of the grid sums chunks
      named_bar_sync(1, kConsumerThreads);
      if (threadIdx.x == 0) grid_barrier(prm.barrier);
      named_bar_sync(1, kConsumerThreads);
      norm_finish_all(prm.norms, (int)blockIdx.x * (kConsumerThreads / 32) + warp, (int)gridDim.x * (kConsumerThreads / 32));
    }
  }
  __syncthreads();
  stamp(3);
}

}  // namespace gaccum
