/* CPU oracle (plain C + OpenMP, fp32) for the gradient-accumulation train_op.
 *
 * TEST INFRASTRUCTURE ONLY -- never linked into or loaded by the shipped library.  Users:
 * tests/, __graft_entry__.smoke(), and bench.py's cpu_baseline / --impl reference legs.
 *
 * PARITY STATUS: same as oracle/oracle_np.py -- pinned against the reference's own
 * optimization.py executed over oracle/tf_stub (tests/golden) and against hand-derived
 * known answers; the TF primitives' semantics are restated from TF 1.15 and are NOT pinned
 * by a real TensorFlow run ("parity unpinned" at that level).
 *
 * Structure mirrors the reference's UN-FUSED graph on purpose: one loop per TF op, every
 * intermediate materialised, because this file is also the stopwatch for "the reference's
 * CPU path" (all host cores via OpenMP, as TF's Eigen pool would use).
 * Citations are relative to the reference repository's root.
 * Build: see oracle/Makefile (gcc -O2 -ffp-contract=off -fopenmp -shared -fPIC).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#define ORACLE_API __attribute__((visibility("default")))

typedef struct {
  int32_t variant;            /* 0 = AdamWeightDecayOptimizer (optimization.py:107), 1 = tf.train.AdamOptimizer */
  int32_t _pad;
  /* Python floats are doubles; the reference converts them to fp32 at different points
   * (e.g. (1.0 - beta_1) is evaluated in double first, optimization.py:152), so keep doubles. */
  double beta1, beta2, epsilon, weight_decay_rate, clip_norm;
} oracle_hparams;

/* ---- a2: LR schedule, optimization.py:29-54 (fp32 op order of TF 1.15 PolynomialDecay) ---- */
ORACLE_API float oracle_learning_rate(double init_lr, int64_t num_train_steps,
                                      int64_t num_warmup_steps, int64_t global_step) {
  volatile float lr0 = (float)init_lr;                 /* :29 */
  volatile float gs = (float)global_step;              /* cast(step, f32) */
  volatile float ds = (float)num_train_steps;
  if (gs > ds) gs = ds;                                /* minimum(gs, decay_steps) */
  volatile float p = gs / ds;
  volatile float omp = 1.0f - p;
  volatile float lr = lr0 * omp;                       /* (lr0-0)*pow(1-p,1)+0 */
  if (num_warmup_steps) {                              /* :42 */
    int32_t gi = (int32_t)global_step, wi = (int32_t)num_warmup_steps;   /* :43-44 */
    volatile float pct = (float)gi / (float)wi;        /* :46-49 */
    volatile float wlr = (float)init_lr * pct;         /* :50 */
    volatile float isw = gi < wi ? 1.0f : 0.0f;        /* :52 */
    volatile float a = (1.0f - isw) * lr;
    volatile float b = isw * wlr;
    lr = a + b;                                        /* :53-54 */
  }
  return lr;
}

/* ---- a6: assign_add, optimization.py:81,93 ---- */
ORACLE_API void oracle_assign_add(float* a, const float* g, int64_t n) {
#pragma omp parallel for schedule(static) if (n > 16384)
  for (int64_t i = 0; i < n; ++i) a[i] = a[i] + g[i];
}

/* un-fused elementwise helpers: each is one TF op with a materialised output */
static void op_mul_s(float* o, float s, const float* x, int64_t n) {
#pragma omp parallel for schedule(static) if (n > 16384)
  for (int64_t i = 0; i < n; ++i) o[i] = s * x[i];
}
static void op_div_s(float* o, const float* x, float s, int64_t n) {
#pragma omp parallel for schedule(static) if (n > 16384)
  for (int64_t i = 0; i < n; ++i) o[i] = x[i] / s;
}
static void op_add(float* o, const float* x, const float* y, int64_t n) {
#pragma omp parallel for schedule(static) if (n > 16384)
  for (int64_t i = 0; i < n; ++i) o[i] = x[i] + y[i];
}
static void op_sub(float* o, const float* x, const float* y, int64_t n) {
#pragma omp parallel for schedule(static) if (n > 16384)
  for (int64_t i = 0; i < n; ++i) o[i] = x[i] - y[i];
}
static void op_mul(float* o, const float* x, const float* y, int64_t n) {
#pragma omp parallel for schedule(static) if (n > 16384)
  for (int64_t i = 0; i < n; ++i) o[i] = x[i] * y[i];
}
static void op_div(float* o, const float* x, const float* y, int64_t n) {
#pragma omp parallel for schedule(static) if (n > 16384)
  for (int64_t i = 0; i < n; ++i) o[i] = x[i] / y[i];
}
static void op_sqrt(float* o, const float* x, int64_t n) {
#pragma omp parallel for schedule(static) if (n > 16384)
  for (int64_t i = 0; i < n; ++i) o[i] = sqrtf(x[i]);
}
static void op_add_s(float* o, const float* x, float s, int64_t n) {
#pragma omp parallel for schedule(static) if (n > 16384)
  for (int64_t i = 0; i < n; ++i) o[i] = x[i] + s;
}

/* l2_loss(x) = sum(x^2)/2, defined as the correctly-rounded sum (fp64 accumulation in fixed
 * 4096-element blocks so the value does not depend on the thread count), one rounding to fp32. */
#define L2_BLOCK 4096
ORACLE_API float oracle_l2_loss(const float* x, int64_t n) {
  int64_t nb = (n + L2_BLOCK - 1) / L2_BLOCK;
  double* part = (double*)malloc(sizeof(double) * (size_t)(nb > 0 ? nb : 1));
#pragma omp parallel for schedule(static) if (n > 16384)
  for (int64_t b = 0; b < nb; ++b) {
    int64_t lo = b * L2_BLOCK, hi = lo + L2_BLOCK < n ? lo + L2_BLOCK : n;
    double s = 0.0;
    for (int64_t i = lo; i < hi; ++i) s += (double)x[i] * (double)x[i];
    part[b] = s;
  }
  double s = 0.0;
  for (int64_t b = 0; b < nb; ++b) s += part[b];
  free(part);
  return (float)(s / 2.0);
}

/* a8: tf.clip_by_global_norm scale (TF 1.15): clip*min(1/gn, 1/clip) + (gn-gn) */
ORACLE_API float oracle_clip_scale(float gn, float clip) {
  volatile float inv = 1.0f / gn;
  volatile float invc = 1.0f / clip;
  volatile float mn = inv < invc ? inv : invc;         /* Minimum: NaN handled below */
  if (inv != inv) mn = inv;
  volatile float s = clip * mn;
  volatile float z = gn - gn;
  return s + z;
}

/* One micro-step.  params/grads/accum/m/v: arrays of T per-tensor pointers (grads[i] may be NULL).
 * scratch: caller-provided fp32 buffer of at least 6*max(numel) elements.
 * beta_pow: {beta1_power, beta2_power} for variant 1 (updated on apply, TF1 Adam._finish).
 * out_info: {applied, lr, global_norm, clip_scale}.  Returns 0, or -1 on bad args. */
ORACLE_API int oracle_step(int32_t T, const int64_t* numel, float* const* params,
                           const float* const* grads, float* const* accum, float* const* m,
                           float* const* v, const uint8_t* decay, const oracle_hparams* hp,
                           int64_t global_step, int32_t N, float lr, float* beta_pow,
                           float* scratch, float* out_info) {
  if (T < 0 || N <= 0 || !hp) return -1;
  int is_apply = ((int32_t)global_step % N) == 0;      /* optimization.py:77,91 */
  for (int32_t t = 0; t < T; ++t)                      /* :81 / :93 */
    if (grads[t]) oracle_assign_add(accum[t], grads[t], numel[t]);
  float gn = 0.0f, scale = 1.0f;
  if (is_apply) {
    const float nf = (float)N;
    int64_t mx = 0;
    for (int32_t t = 0; t < T; ++t) if (numel[t] > mx) mx = numel[t];
    float *t0 = scratch, *t1 = scratch + mx, *t2 = scratch + 2 * mx, *t3 = scratch + 3 * mx,
          *t4 = scratch + 4 * mx, *t5 = scratch + 5 * mx;
    int do_clip = hp->clip_norm > 0.0;
    if (do_clip) {                                     /* :83-84, global norm over ALL tensors first */
      volatile float half = 0.0f;
      for (int32_t t = 0; t < T; ++t) {
        op_mul_s(t0, 1.0f, accum[t], numel[t]);
        op_div_s(t1, t0, nf, numel[t]);
        half = half + oracle_l2_loss(t1, numel[t]);
      }
      volatile float two = half * 2.0f;
      gn = sqrtf(two);
      scale = oracle_clip_scale(gn, (float)hp->clip_norm);
    }
    const float b1 = (float)hp->beta1, b2 = (float)hp->beta2, eps = (float)hp->epsilon,
                wd = (float)hp->weight_decay_rate;
    volatile float alpha = 0.0f;
    volatile float omb1, omb2;
    if (hp->variant == 0) {
      omb1 = (float)(1.0 - hp->beta1);                 /* :152 -- Python double, then fp32 */
      omb2 = (float)(1.0 - hp->beta2);                 /* :154 */
    } else {
      omb1 = 1.0f - b1; omb2 = 1.0f - b2;              /* ApplyAdam: T(1) - beta1() in fp32 */
      volatile float s1 = 1.0f - beta_pow[1];
      volatile float s2 = sqrtf(s1);
      volatile float s3 = lr * s2;
      volatile float s4 = 1.0f - beta_pow[0];
      alpha = s3 / s4;
    }
    for (int32_t t = 0; t < T; ++t) {
      const int64_t n = numel[t];
      float* c = t1;
      op_mul_s(t0, 1.0f, accum[t], n);                 /* :83 */
      op_div_s(t1, t0, nf, n);
      if (do_clip) { op_mul_s(t0, scale, t1, n); c = t0; }   /* :84 values * scale */
      if (hp->variant == 0) {                          /* optimization.py:151-176 */
        float* nm = t2; float* nv = t3;
        op_mul_s(t4, b1, m[t], n); op_mul_s(t5, omb1, c, n); op_add(nm, t4, t5, n);      /* :151-152 */
        op_mul(t4, c, c, n); op_mul_s(t5, omb2, t4, n); op_mul_s(t4, b2, v[t], n);
        op_add(nv, t4, t5, n);                                                            /* :153-155 */
        op_sqrt(t4, nv, n); op_add_s(t5, t4, eps, n); op_div(t4, nm, t5, n);             /* :157 */
        if (decay[t]) { op_mul_s(t5, wd, params[t], n); op_add(t4, t4, t5, n); }         /* :166-167 */
        op_mul_s(t5, lr, t4, n);                                                          /* :169 */
        op_sub(params[t], params[t], t5, n);                                              /* :171,174 */
        memcpy(m[t], nm, sizeof(float) * (size_t)n);                                      /* :175 */
        memcpy(v[t], nv, sizeof(float) * (size_t)n);                                      /* :176 */
      } else {                                         /* TF1 ApplyAdam */
        op_sub(t2, c, m[t], n); op_mul_s(t3, omb1, t2, n); op_add(m[t], m[t], t3, n);
        op_mul(t2, c, c, n); op_sub(t3, t2, v[t], n); op_mul_s(t2, omb2, t3, n); op_add(v[t], v[t], t2, n);
        op_mul_s(t2, alpha, m[t], n); op_sqrt(t3, v[t], n); op_add_s(t4, t3, eps, n);
        op_div(t3, t2, t4, n); op_sub(params[t], params[t], t3, n);
      }
    }
    if (hp->variant == 1) {
      volatile float p1 = beta_pow[0] * b1, p2 = beta_pow[1] * b2;
      beta_pow[0] = p1; beta_pow[1] = p2;
    }
    for (int32_t t = 0; t < T; ++t)                    /* :86-87 */
      memset(accum[t], 0, sizeof(float) * (size_t)numel[t]);
  }
  if (out_info) { out_info[0] = (float)is_apply; out_info[1] = lr; out_info[2] = gn; out_info[3] = scale; }
  return 0;
}

ORACLE_API void oracle_set_num_threads(int n) {
#ifdef _OPENMP
  if (n > 0) omp_set_num_threads(n);
#else
  (void)n;
#endif
}

ORACLE_API int oracle_num_threads(void) {
  int n = 1;
#ifdef _OPENMP
#pragma omp parallel
  {
#pragma omp master
    n = omp_get_num_threads();
  }
#endif
  return n;
}
