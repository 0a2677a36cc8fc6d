// gaccum_lamb.cuh -- the apply step of GACCUM_LAMB (include/gaccum.h; You et al. 2019, in TF-Addons' form).
//
// LAMB scales each tensor's update by its trust ratio r = ||p|| / ||u||, so a tensor can only be written once the
// norms of ALL its tiles are known -- a per-tensor reduction after the global-norm one.  One cooperative launch of
// kLambBlocksPerSm x 256-thread CTAs per SM, each owning a contiguous range of the tile table, in three phases:
//
//   phase 1  (clipping or loss scaling only)  a' = a + G, stored back; the global norm of a'/N (of (a'/N)/S loss-scaled)
//            and the non-finite flag, in the launch's exact accumulator (LaunchCounters, as apply_clip_kernel does)
//   barrier  every CTA derives the same clip scale s and the same skip decision (window_decision)
//   phase 2  read a' (a + G without phase 1), p, m, v; store m, v and the update u -- into the accumulator slab, in place
//            of a'.  Each tile's sum(p^2) and sum(u^2) go exactly into per-tensor accumulators: per-warp fp64 partials
//            into the CTA's per-warp fixed-point bins, flushed (integer atomics) when the CTA's next tile belongs to
//            another tensor -- the sums do not depend on which CTA reduced which tile
//   barrier  one warp per tensor turns its two sums into r, stored in the plan's ratio array
//   barrier
//   phase 3  read p and u, store p - (r*lr_t)*u (fp32, or the master weights plus their RNE model copy) and a = +0;
//            lr_t = lr * mult[t], the tensor's learning-rate multiplier (LrMultParams), read once per tile
//
// A skipped window (loss scaling) runs neither phase 2 nor the ratio step: it stores a = +0 and nothing else, so the
// ratios of the last applied window stay.  Bytes: phase 2 reads a', p, m, v (and G) and writes m, v, u; phase 3 reads
// p, u and writes p, a: 48 B/param (gaccum_algorithmic_bytes), plus the a' round trip of phase 1.
//
// Per-launch state: the LaunchCounters of the clip-apply and, per tensor, a LambTensorAcc -- both in two sets, launch
// k using set k & 1 (k read off the plan's monotonic barrier counter) and clearing the other: no host-side state, so
// launches replay in CUDA graphs.
#pragma once

#include "gaccum_kernels.cuh"

namespace gaccum {

constexpr int kLambBlocksPerSm = 3;

// sum(p^2) and sum(u^2) of one tensor in one launch, exact (acc_add); nonfinite as LaunchCounters::nonfinite bits 0-1
struct LambTensorAcc {
  unsigned long long bins[2][kAccBins];
  unsigned int nonfinite[2];
  unsigned int pad[2];
};
static_assert(sizeof(LambTensorAcc) % 8 == 0, "cleared in 8-byte words");

// what phase 2 needs besides Scalars: the clip scale, 1/S, and the bias corrections 1 - beta^t
struct LambCoef {
  float s, inv_s, omb1p, omb2p;
};

// m, v and the update u of one element (gaccum.h, GACCUM_LAMB): one correctly rounded op per TF op
__device__ __forceinline__ float lamb_u(float c, float p, float& m, float& v, bool decay, const Scalars& sc, const LambCoef& k) {
  m = __fadd_rn(__fmul_rn(sc.b1, m), __fmul_rn(sc.omb1, c));
  v = __fadd_rn(__fmul_rn(sc.b2, v), __fmul_rn(sc.omb2, __fmul_rn(c, c)));
  const float mh = __fdiv_rn(m, k.omb1p);
  const float vh = __fdiv_rn(v, k.omb2p);
  float u = __fdiv_rn(mh, __fadd_rn(__fsqrt_rn(vh), sc.eps));
  if (decay) u = __fadd_rn(u, __fmul_rn(sc.wd, p));
  return u;
}
__device__ __forceinline__ double add_sq64(double acc, float x) { return fma((double)x, (double)x, acc); }
__device__ __forceinline__ double add_sq64(double acc, const float4 x) {
  return add_sq64(add_sq64(add_sq64(add_sq64(acc, x.x), x.y), x.z), x.w);
}

// ---- phase 1: a' = a + G stored back; returns this thread's fp32 partial of the global norm (as norm_tile) ----
// norms (kLsNoClip only; launch-uniform): the partial of sum(((a'/N)(1/S))^2) is formed as kLsClip forms it.
template <int MODE, bool H, int CAP>
__device__ __forceinline__ float lamb_norm_tile(const TileDesc& d, const KernelParams<CAP>& prm, const float inv_s, bool& bad,
                                                const Divisor& dv, const bool norms) {
  const Grad<H> g(prm, d);
  float* __restrict__ a = prm.accum + (size_t)d.soff32 * kSlabAlign;
  float4* a4 = reinterpret_cast<float4*>(a);
  float acc = 0.f;
  float4 x[kUnroll], gg[kUnroll];
  walk_tile(d.len, (g.g == nullptr || g.vec_ok()) ? d.len >> 2 : 0u, threadIdx.x,
            [&](int u, uint32_t i) { x[u] = a4[i]; if (g.g) gg[u] = g.vec(i); },
            [] {},
            [&](int u, uint32_t i) {
              if (g.g) { x[u] = add_rn(x[u], gg[u]); a4[i] = x[u]; }
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

// ---- phase 2: m, v and u of one tile (u into the accumulator slab); this thread's sums of p^2 and u^2 ----
// LOAD_G: there was no phase 1, so a' = a + G is formed here, and with norms (launch-uniform) the thread's fp32 partial of
// sum((a'/N)^2) goes into sg.  H: p is the master slab.
template <int MODE, bool LOAD_G, bool H, int CAP>
__device__ __forceinline__ void lamb_update_tile(const TileDesc& d, const KernelParams<CAP>& prm, const LambCoef& k,
                                                 const Divisor& dv, double& sp, double& su, const bool norms, float& sg) {
  Grad<H> g;
  if constexpr (LOAD_G) g = Grad<H>(prm, d);
  const size_t soff = (size_t)d.soff32 * kSlabAlign;
  float* __restrict__ a = prm.accum + soff;
  float* __restrict__ m = prm.m + soff;
  float* __restrict__ v = prm.v + soff;
  const float* __restrict__ p = update_ptr<H>(prm, d);
  const bool decay = (d.tensor_flags >> 31) != 0;
  const Scalars& sc = prm.sc;
  float4* a4 = reinterpret_cast<float4*>(a);
  float4* m4 = reinterpret_cast<float4*>(m);
  float4* v4 = reinterpret_cast<float4*>(v);
  const float4* p4 = reinterpret_cast<const float4*>(p);
  float4 va[kUnroll], vg[kUnroll], vp[kUnroll], vm[kUnroll], vv[kUnroll];
  walk_tile(d.len, (H || aligned16(p)) && (g.g == nullptr || g.vec_ok()) ? d.len >> 2 : 0u, threadIdx.x,
            [&](int u, uint32_t i) {
              va[u] = a4[i]; vp[u] = __ldcs(p4 + i); vm[u] = __ldcs(m4 + i); vv[u] = __ldcs(v4 + i);
              if (LOAD_G && g.g) vg[u] = g.vec(i);
            },
            [] {},
            [&](int u, uint32_t i) {
              if (LOAD_G && g.g) va[u] = add_rn(va[u], vg[u]);
              if (LOAD_G && norms) sg = add_sq(sg, va[u], dv);
              float4 w;
              w.x = lamb_u(mode_c<MODE>(va[u].x, k.s, k.inv_s, dv), vp[u].x, vm[u].x, vv[u].x, decay, sc, k);
              w.y = lamb_u(mode_c<MODE>(va[u].y, k.s, k.inv_s, dv), vp[u].y, vm[u].y, vv[u].y, decay, sc, k);
              w.z = lamb_u(mode_c<MODE>(va[u].z, k.s, k.inv_s, dv), vp[u].z, vm[u].z, vv[u].z, decay, sc, k);
              w.w = lamb_u(mode_c<MODE>(va[u].w, k.s, k.inv_s, dv), vp[u].w, vm[u].w, vv[u].w, decay, sc, k);
              __stcs(m4 + i, vm[u]); __stcs(v4 + i, vv[u]); a4[i] = w;
              sp = add_sq64(sp, vp[u]); su = add_sq64(su, w);
            },
            [&](uint32_t i) {
              float ax = a[i], mx = m[i], vx = v[i];
              const float px = p[i];
              if (LOAD_G && g.g) ax = __fadd_rn(ax, g.elem(i));
              if (LOAD_G && norms) sg = add_sq(sg, ax, dv);
              const float w = lamb_u(mode_c<MODE>(ax, k.s, k.inv_s, dv), px, mx, vx, decay, sc, k);
              m[i] = mx; v[i] = vx; a[i] = w;
              sp = add_sq64(sp, px); su = add_sq64(su, w);
            });
}

// ---- phase 3: p = p - (r*lr)*u and a = +0 (a = +0 only on a skipped window) ----
// Deferred reset (DeferredResetParams): a = +0 is not stored, and the u lines read are discarded from L2.
// EMA: e is read with p and u, and e - (e - p) * c stored after p.
// norms (launch-uniform): the thread's fp32 partials of p^2 (p before the update; on a skipped window p is read for it)
// and (p - p')^2 go into nw and nu.
template <bool H, int CAP, bool EMA = false>
__device__ __forceinline__ void lamb_write_tile(const TileDesc& d, const KernelParams<CAP>& prm, const float rlr, const bool write,
                                                const bool norms, float& nw, float& nu, float* ema = nullptr,
                                                const float ema_c = 0.f) {
  const size_t soff = (size_t)d.soff32 * kSlabAlign;
  float* __restrict__ a = prm.accum + soff;
  float* __restrict__ p = update_ptr<H>(prm, d);
  float* __restrict__ e = EMA ? ema + soff : nullptr;
  uint16_t* q = nullptr;
  bool bf16 = false;
  if constexpr (H) { q = model_ptr(prm, d); bf16 = prm.half.bf16 != 0; }
  const bool deferred = prm.dr.accum_zero != nullptr;   // launch-uniform: a = +0 is not stored (DeferredResetParams)
  float4* a4 = reinterpret_cast<float4*>(a);
  float4* p4 = reinterpret_cast<float4*>(p);
  float4* e4 = reinterpret_cast<float4*>(e);
  float4 vu[kUnroll], vp[kUnroll], ve[kUnroll];
  const uint32_t nvec = H || aligned16(p) ? d.len >> 2 : 0u;
  walk_tile(d.len, nvec, threadIdx.x,
            [&](int u, uint32_t i) {
              if (write) {
                vu[u] = __ldcs(a4 + i); vp[u] = __ldcs(p4 + i);
                if constexpr (EMA) ve[u] = __ldcs(e4 + i);
              } else if (norms) {
                vp[u] = __ldcs(p4 + i);
              }
            },
            [] {},
            [&](int u, uint32_t i) {
              if (write) {
                const float4 pb = vp[u];
                vp[u].x = __fsub_rn(vp[u].x, __fmul_rn(rlr, vu[u].x));
                vp[u].y = __fsub_rn(vp[u].y, __fmul_rn(rlr, vu[u].y));
                vp[u].z = __fsub_rn(vp[u].z, __fmul_rn(rlr, vu[u].z));
                vp[u].w = __fsub_rn(vp[u].w, __fmul_rn(rlr, vu[u].w));
                if (norms) {
                  nw = sq_acc(nw, pb);
                  nu = diff_sq_acc(diff_sq_acc(diff_sq_acc(diff_sq_acc(nu, pb.x, vp[u].x), pb.y, vp[u].y), pb.z, vp[u].z),
                                   pb.w, vp[u].w);
                }
                __stcs(p4 + i, vp[u]);
                if constexpr (H) store_model4(q, i, vp[u], bf16);
                if constexpr (EMA) __stcs(e4 + i, ema_vec(ve[u], vp[u], ema_c));
              } else if (norms) {
                nw = sq_acc(nw, vp[u]);
              }
              if (!deferred) __stcs(a4 + i, make_float4(0.f, 0.f, 0.f, 0.f));   // optimization.py:86-87
            },
            [&](uint32_t i) {
              if (write) {
                const float pb = p[i];
                const float px = __fsub_rn(pb, __fmul_rn(rlr, a[i]));
                if (norms) { nw = sq_acc(nw, pb); nu = diff_sq_acc(nu, pb, px); }
                p[i] = px;
                if constexpr (H) q[i] = (uint16_t)f2h(px, bf16);
                if constexpr (EMA) e[i] = ema_elem(e[i], px, ema_c);
              } else if (norms) {
                nw = sq_acc(nw, p[i]);
              }
              if (!deferred) a[i] = 0.f;
            });
  if (deferred) {
    // the u lines are dead once read: a line is vectors 8l .. 8l + 7, which 8 lanes of one warp have loaded and used by
    // now; whole vector lines only (a tail line holds elements other threads read)
    __syncwarp();
    const uint32_t tid = threadIdx.x;
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      const uint32_t i = u * kThreads + tid;
      if ((tid & 7u) == 0u && i + 8u <= nvec) discard_line(a4 + i);
    }
  }
}

// Device state (loss scaling, EMA, window weight, device schedule): thread 0 of every CTA reads it during set-up
// (launch_begin); block 0's thread 0 commits the launch at the very end, past the grid barriers (launch_commit).
template <int CAP, int MODE, bool H = false, bool EMA = false>
__global__ void __launch_bounds__(kThreads, kLambBlocksPerSm)
lamb_apply_kernel(const __grid_constant__ KernelParams<CAP> prm) {
  constexpr bool kPhase1 = MODE != kNoClip;
  const bool norms = prm.norms.out != nullptr;   // launch-uniform: one more grid barrier at the end of the launch
  const unsigned long long kBarriers = (kPhase1 ? 3 : 2) + (norms ? 1 : 0);
  constexpr int kWarps = kThreads / 32;
  const LambParams& lb = prm.lamb;
  __shared__ unsigned long long s_bins[kWarps][2][kAccBins];   // one pair of exact accumulators per warp (8.5 KB)
  __shared__ unsigned int s_nonfinite[2];
  __shared__ float s_bcast[2];
  __shared__ LaunchStep<EMA> s_step;
  __shared__ LossScaleState s_ls;        // loss-scaled: the state as this launch found it
  __shared__ int s_skip;
  __shared__ uint32_t s_set;

  const int warp = (int)threadIdx.x >> 5, lane = (int)threadIdx.x & 31;
  const int nt = prm.num_tiles;
  const int t_lo = (int)((long long)nt * blockIdx.x / gridDim.x);      // this CTA's tiles [t_lo, t_hi)
  const int t_hi = (int)((long long)nt * (blockIdx.x + 1) / gridDim.x);

  if (threadIdx.x == 0) {
    // every CTA that has not yet arrived at this launch's first barrier reads a value in [k*B*grid, (k*B+1)*grid)
    const unsigned long long k = ld_acquire_gpu_u64(prm.barrier) / ((unsigned long long)gridDim.x * kBarriers);
    s_set = (uint32_t)(k & 1ull);
    s_nonfinite[0] = s_nonfinite[1] = 0;
    s_bcast[0] = 1.f;
    s_bcast[1] = 0.f;
    s_skip = 0;
    launch_begin<kLamb, MODE, EMA>(prm, s_step, &s_ls);
  }
  for (int i = threadIdx.x; i < kWarps * 2 * kAccBins; i += kThreads) (&s_bins[0][0][0])[i] = 0ull;
  __syncthreads();
  // device schedule: every CTA read the same step, so all of them leave here or none does (before any barrier)
  if (!s_step.ok) { sched_refuse(prm.sched); return; }
  const uint32_t set = s_set;
  // the launch's divisor, held in registers: read from shared memory at every use it slowed the unweighted apply 1.6-2.2 %
  const Divisor dv = s_step.dv;
  LaunchCounters* const ctr = prm.counters + set;
  LambTensorAcc* const tacc = lb.acc + (size_t)set * lb.num_tensors;
  clear_other_counters(prm.counters, set);
  {
    unsigned long long* other = reinterpret_cast<unsigned long long*>(lb.acc + (size_t)(set ^ 1u) * lb.num_tensors);
    const size_t words = (size_t)lb.num_tensors * (sizeof(LambTensorAcc) / 8);
    for (size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x; i < words; i += (size_t)gridDim.x * kThreads) other[i] = 0ull;
  }
  // the step's lr and beta powers, held in registers from set-up on: read from shared memory where phases 2 and 3 use
  // them, the 16-bit kLsNoClip instantiations spill more
  const float lr = s_step.lr, b1p = s_step.b1p, b2p = s_step.b2p;
  float inv_s = 1.0f;
  if constexpr (loss_scaled(MODE)) inv_s = __fdiv_rn(1.0f, s_ls.scale);   // exact: S is a power of two

  // ---- phase 1: a' and the global norm ----
  if constexpr (kPhase1) {
    bool bad = false;
    unsigned int nonfinite = 0;
    for (int t = t_lo; t < t_hi; ++t) {
      const float part = lamb_norm_tile<MODE, H>(prm.tiles[t], prm, inv_s, bad, dv, norms);
      if (MODE != kLsNoClip || norms) {
        const double w = warp_sum((double)part);
        if (lane == 0) {
          if constexpr (MODE != kLsNoClip) acc_add(s_bins[warp][0], nonfinite, w);
          if (norms) prm.norms.tile_part[((size_t)t * kNormCols) * kNormWarps + warp] = w;
        }
      }
    }
    if constexpr (loss_scaled(MODE)) { if (bad) nonfinite |= kElemNonfinite; }
    if (nonfinite) atomicOr(&s_nonfinite[0], nonfinite);
    __syncthreads();
    if (threadIdx.x < kAccBins) {
      unsigned long long v = 0;
      for (int w = 0; w < kWarps; ++w) { v += s_bins[w][0][threadIdx.x]; s_bins[w][0][threadIdx.x] = 0ull; }
      if (v) atomicAdd(&ctr->bins[threadIdx.x], v);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      if (s_nonfinite[0]) atomicOr(&ctr->nonfinite, s_nonfinite[0]);
      s_nonfinite[0] = 0;
      grid_barrier(prm.barrier);
    }
    __syncthreads();
    if constexpr (MODE != kLsNoClip) {
      if (threadIdx.x < kAccBins) s_bins[0][1][threadIdx.x] = __ldcg(&ctr->bins[threadIdx.x]);
      __syncthreads();
    }
    if (threadIdx.x == 0) window_decision<MODE>(ctr, s_bins[0][1], prm.sc.clip, s_bcast[0], s_bcast[1], s_skip);
    __syncthreads();
    if (threadIdx.x < kAccBins) s_bins[0][1][threadIdx.x] = 0ull;
    __syncthreads();
  }
  const bool skip = s_skip != 0;
  const LambCoef coef{s_bcast[0], inv_s, __fsub_rn(1.0f, b1p), __fsub_rn(1.0f, b2p)};

  // ---- phase 2: m, v, u and the per-tensor sums ----
  if (!skip) {
    int cur = -1;
    bool cur_adapt = false;
    auto flush = [&] {                                      // the CTA's sums of tensor `cur` -> its global accumulators
      __syncthreads();
      if (threadIdx.x < 2 * kAccBins) {
        const int which = (int)threadIdx.x / kAccBins, i = (int)threadIdx.x % kAccBins;
        unsigned long long v = 0;
        for (int w = 0; w < kWarps; ++w) { v += s_bins[w][which][i]; s_bins[w][which][i] = 0ull; }
        if (v) atomicAdd(&tacc[cur].bins[which][i], v);
      }
      if (threadIdx.x < 2 && s_nonfinite[threadIdx.x]) {
        atomicOr(&tacc[cur].nonfinite[threadIdx.x], s_nonfinite[threadIdx.x]);
        s_nonfinite[threadIdx.x] = 0;
      }
      __syncthreads();
    };
    for (int t = t_lo; t < t_hi; ++t) {
      const TileDesc d = prm.tiles[t];
      const int ti = (int)(d.tensor_flags & 0x7fffffffu);
      if (ti != cur) {
        if (cur_adapt) flush();
        cur = ti;
        cur_adapt = lb.adapt[ti] != 0;
      }
      double sp = 0.0, su = 0.0;
      float sg = 0.f;
      lamb_update_tile<MODE, !kPhase1, H>(d, prm, coef, dv, sp, su, norms, sg);
      if (!kPhase1 && norms) norm_store(prm.norms, t, 0, warp, sg);
      if (cur_adapt) {
        sp = warp_sum(sp);
        su = warp_sum(su);
        if (lane == 0) {
          unsigned int nfp = 0, nfu = 0;
          acc_add(s_bins[warp][0], nfp, sp);
          acc_add(s_bins[warp][1], nfu, su);
          if (nfp) atomicOr(&s_nonfinite[0], nfp);
          if (nfu) atomicOr(&s_nonfinite[1], nfu);
        }
      }
    }
    if (cur_adapt) flush();
  }
  __syncthreads();
  if (threadIdx.x == 0) grid_barrier(prm.barrier);
  __syncthreads();

  // ---- trust ratios: one warp per tensor, r = ||p|| / ||u|| from the exact sums ----
  if (!skip) {
    for (int ti = (int)blockIdx.x * kWarps + warp; ti < lb.num_tensors; ti += (int)gridDim.x * kWarps) {
      float r = 1.0f;
      if (lb.adapt[ti]) {
        unsigned long long* bins = &s_bins[warp][0][0];
        for (int i = lane; i < 2 * kAccBins; i += 32) bins[i] = __ldcg(&tacc[ti].bins[0][0] + i);
        __syncwarp();
        if (lane == 0) {
          const float wn = __fsqrt_rn((float)acc_value(s_bins[warp][0], __ldcg(&tacc[ti].nonfinite[0])));
          const float un = __fsqrt_rn((float)acc_value(s_bins[warp][1], __ldcg(&tacc[ti].nonfinite[1])));
          r = (wn > 0.f && un > 0.f) ? __fdiv_rn(wn, un) : 1.0f;
        }
        __syncwarp();
      }
      if (lane == 0) lb.ratios[ti] = r;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) grid_barrier(prm.barrier);
  __syncthreads();

  // ---- phase 3: the parameters and a = +0 ----
  for (int t = t_lo; t < t_hi; ++t) {
    const TileDesc d = prm.tiles[t];
    // ratio * lr_t first, lr_t = lr * mult[t] (LrMultParams)
    const float rlr = skip ? 0.f : __fmul_rn(__ldcg(&lb.ratios[d.tensor_flags & 0x7fffffffu]),
                                             tile_rate<0>(lr, tensor_mult(prm.lrm, d), 0.f, 1.f));
    float nw = 0.f, nu = 0.f;
    if constexpr (EMA) lamb_write_tile<H, CAP, true>(d, prm, rlr, !skip, norms, nw, nu, prm.ema.slab, s_step.ema.c);
    else lamb_write_tile<H>(d, prm, rlr, !skip, norms, nw, nu);
    if (norms) {
      norm_store(prm.norms, t, 1, warp, nw);
      norm_store(prm.norms, t, 2, warp, nu);
    }
  }

  if (blockIdx.x == 0 && threadIdx.x == 0) launch_commit<kLamb, MODE, EMA>(prm, s_step, &s_ls, skip, s_bcast[1], s_bcast[0]);
  if (norms) {
    // every tile's partials are stored once every CTA is through phase 3: one more grid barrier, then every warp of
    // the grid sums chunks
    __syncthreads();
    if (threadIdx.x == 0) grid_barrier(prm.barrier);
    __syncthreads();
    norm_finish_all(prm.norms, (int)blockIdx.x * kWarps + warp, (int)gridDim.x * kWarps);
  }
}

}  // namespace gaccum
