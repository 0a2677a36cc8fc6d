// gaccum_tf_op.cc -- the `tf.load_op_library` custom ops that put libgaccum.so behind the
// reference's unchanged `create_optimizer(...)` (reference optimization.py:25-104).
//
// NOT BUILT AGAINST TENSORFLOW IN THIS REPOSITORY'S IMAGE: TensorFlow (headers and runtime) is absent here
// (DESIGN.md "Boundary").  What IS exercised here: this file, unmodified, compiled against a mock of the op-kernel
// API it uses (tests/tf_mock) and driven by tests/tf_mock/tf_op_driver.cc -- registration, attribute parsing, input
// indexing, ref / resource variables, HostMemory scalars, error paths on CPU; Compute() -> gaccum_step -> the CUDA
// kernels against the reference's fixtures on the GPU (tests/test_tf_op_adapter.py); and the Python half of the
// shim over an emulated op (tests/test_tf_shim_stub.py).  Build where TensorFlow >= 2.11 with tf.compat.v1 exists
// (se::Stream::platform_specific_handle(); older releases spell it stream->implementation()->GpuStreamHack()):
//
//   TF_CFLAGS=$(python -c 'import tensorflow as tf; print(" ".join(tf.sysconfig.get_compile_flags()))')
//   TF_LFLAGS=$(python -c 'import tensorflow as tf; print(" ".join(tf.sysconfig.get_link_flags()))')
//   g++ -std=c++17 -shared -fPIC gaccum_tf_op.cc -o libgaccum_tf.so $TF_CFLAGS $TF_LFLAGS \
//       -I../../include -L../csrc -lgaccum -Wl,-rpath,'$ORIGIN/../csrc' -DGOOGLE_CUDA=1
//
// Two registrations of the same adapter, differing only in how the variables arrive:
//   GaccumStep    params: N * Ref(float), accum / m / v: Ref(float)        TF1 ref variables (run_classifier.py under TF 1.x)
//   GaccumStepV2  params: N * resource,   accum / m / v: resource           resource variables (what Keras layers create in
//                                                                           distributedExample/02, 04 under TF >= 2)
// Common inputs: grads: N * float, global_step: int64 [host], lr: float [host], beta_powers: float[2] [host]
// Attrs: N, accum_n, variant, decay_mask: list(bool), and the hyper-parameters as STRINGS holding Python's repr() of the
// double: a `float` attr is fp32 in the GraphDef and would lose the reference's double -> fp32 conversion points
// (`1.0 - self.beta_1` is evaluated in double before the cast, optimization.py:152).
//
// The adapter reads raw device pointers and the device stream out of the OpKernelContext and calls gaccum_step
// (include/gaccum.h).  It never allocates device memory, never synchronises, and launches exactly one kernel.
// State (accum/m/v) are ordinary TF variables created by tf_shim/optimization.py, so the Estimator's Saver
// checkpoints them like the reference's per-variable accumulators (optimization.py:78, 137-148) -- as three
// packed tensors instead of 3T.
#include <cstdlib>
#include <string>
#include <vector>

#include "gaccum.h"
#include "tensorflow/core/framework/op.h"
#include "tensorflow/core/framework/op_kernel.h"
#include "tensorflow/core/framework/resource_mgr.h"
#include "tensorflow/core/framework/resource_var.h"
#include "tensorflow/core/framework/shape_inference.h"
#include "tensorflow/core/kernels/training_op_helpers.h"   // PrepareToUpdateVariable
#include "tensorflow/core/platform/stream_executor.h"

namespace tf = tensorflow;

#define GACCUM_COMMON_ATTRS                                    \
  .Input("grads: N * float")                                   \
      .Input("global_step: int64")                             \
      .Input("lr: float")                                      \
      .Input("beta_powers: float")                             \
      .Attr("N: int >= 1")                                     \
      .Attr("accum_n: int >= 1")                               \
      .Attr("variant: int = 0")                                \
      .Attr("beta1: string = '0.9'")                           \
      .Attr("beta2: string = '0.999'")                         \
      .Attr("epsilon: string = '1e-06'")                       \
      .Attr("weight_decay_rate: string = '0.01'")              \
      .Attr("clip_norm: string = '1.0'")                       \
      .Attr("decay_mask: list(bool)")                          \
      .SetIsStateful()                                         \
      .SetShapeFn(tf::shape_inference::NoOutputs)

REGISTER_OP("GaccumStep")
    .Input("params: Ref(N * float)")
    .Input("accum: Ref(float)")
    .Input("m: Ref(float)")
    .Input("v: Ref(float)")
    GACCUM_COMMON_ATTRS.Doc("One micro-step of the gradient-accumulation train_op (reference optimization.py:76-104); ref variables.");

REGISTER_OP("GaccumStepV2")
    .Input("params: N * resource")
    .Input("accum: resource")
    .Input("m: resource")
    .Input("v: resource")
    GACCUM_COMMON_ATTRS.Doc("One micro-step of the gradient-accumulation train_op (reference optimization.py:76-104); resource variables.");

namespace {

// Input order (both ops): params[0..N), accum, m, v, grads[0..N), global_step, lr, beta_powers
template <bool RESOURCE>
class GaccumStepOpT : public tf::OpKernel {
 public:
  explicit GaccumStepOpT(tf::OpKernelConstruction* c) : tf::OpKernel(c) {
    std::string b1, b2, eps, wd, clip;
    OP_REQUIRES_OK(c, c->GetAttr("N", &n_));
    OP_REQUIRES_OK(c, c->GetAttr("accum_n", &accum_n_));
    OP_REQUIRES_OK(c, c->GetAttr("variant", &hp_.variant));
    // the graph op carries no trust-ratio state or adaptation mask: LAMB (variant 2) is a Python train_op feature
    OP_REQUIRES(c, hp_.variant == GACCUM_ADAM_WEIGHT_DECAY || hp_.variant == GACCUM_ADAM,
                tf::errors::InvalidArgument("variant must be 0 (AdamWeightDecay) or 1 (Adam), got ", hp_.variant));
    OP_REQUIRES_OK(c, c->GetAttr("beta1", &b1));
    OP_REQUIRES_OK(c, c->GetAttr("beta2", &b2));
    OP_REQUIRES_OK(c, c->GetAttr("epsilon", &eps));
    OP_REQUIRES_OK(c, c->GetAttr("weight_decay_rate", &wd));
    OP_REQUIRES_OK(c, c->GetAttr("clip_norm", &clip));
    OP_REQUIRES_OK(c, c->GetAttr("decay_mask", &decay_));
    OP_REQUIRES(c, (int)decay_.size() == n_, tf::errors::InvalidArgument("decay_mask must have N entries"));
    hp_.reserved = 0;
    hp_.beta1 = std::strtod(b1.c_str(), nullptr);             // repr(float) round-trips: the exact double Python held
    hp_.beta2 = std::strtod(b2.c_str(), nullptr);
    hp_.epsilon = std::strtod(eps.c_str(), nullptr);
    hp_.weight_decay_rate = std::strtod(wd.c_str(), nullptr);
    hp_.clip_norm = std::strtod(clip.c_str(), nullptr);
  }

  ~GaccumStepOpT() override { gaccum_plan_destroy(plan_); }

  void Compute(tf::OpKernelContext* c) override {
    std::vector<float*> params(n_);
    std::vector<const float*> grads(n_);
    std::vector<int64_t> numels(n_);
    std::vector<tf::core::RefCountPtr<tf::Var>> held;        // resource variables stay alive for the duration of the call
    // The reference relies on control dependencies for ordering (optimization.py:82, 86), not on variable locks:
    // buffers are taken without copy-on-read.  A resource variable whose buffer is shared with a pending read is
    // un-aliased first (PrepareToUpdateVariable), exactly as the built-in ResourceApplyAdam does.
    auto buffer_of = [&](int index, float** ptr, int64_t* numel) -> tf::Status {
      if constexpr (RESOURCE) {
        tf::core::RefCountPtr<tf::Var> var;
        TF_RETURN_IF_ERROR(tf::LookupResource(c, tf::HandleFromInput(c, index), &var));
        tf::mutex_lock ml(*var->mu());
        TF_RETURN_IF_ERROR(tf::PrepareToUpdateVariable<Eigen::GpuDevice, float>(c, var->tensor(), var->copy_on_read_mode.load()));
        *ptr = var->tensor()->flat<float>().data();
        *numel = var->tensor()->NumElements();
        held.push_back(std::move(var));
      } else {
        tf::Tensor t = c->mutable_input(index, /*lock_held=*/true);
        *ptr = t.flat<float>().data();
        *numel = t.NumElements();
      }
      return tf::Status();
    };
    for (int i = 0; i < n_; ++i) {
      OP_REQUIRES_OK(c, buffer_of(i, &params[i], &numels[i]));
      const tf::Tensor& g = c->input(n_ + 3 + i);
      OP_REQUIRES(c, numels[i] == g.NumElements(), tf::errors::InvalidArgument("grad ", i, " does not match its variable"));
      grads[i] = g.flat<float>().data();
    }
    float *accum = nullptr, *m = nullptr, *v = nullptr;
    int64_t n_accum = 0, n_m = 0, n_v = 0;
    OP_REQUIRES_OK(c, buffer_of(n_ + 0, &accum, &n_accum));
    OP_REQUIRES_OK(c, buffer_of(n_ + 1, &m, &n_m));
    OP_REQUIRES_OK(c, buffer_of(n_ + 2, &v, &n_v));
    const int64_t step = c->input(2 * n_ + 3).scalar<int64_t>()();   // HostMemory: the accumulate/apply decision needs no D2H
    const float lr = c->input(2 * n_ + 4).scalar<float>()();          // HostMemory
    auto bp = c->input(2 * n_ + 5).flat<float>();                     // HostMemory

    if (plan_ == nullptr) {   // first run: shapes are static in a TF1 graph
      std::vector<uint8_t> decay(decay_.begin(), decay_.end());
      // the device this kernel was placed on, from TensorFlow -- not from whatever cudaGetDevice() says on this thread
      const auto* info = c->device()->tensorflow_accelerator_device_info();
      OP_REQUIRES(c, info != nullptr, tf::errors::Internal("GaccumStep needs a GPU device (libgaccum has no CPU fallback)"));
      const int dev = info->gpu_id;
      OP_REQUIRES(c, gaccum_plan_create(&plan_, n_, numels.data(), decay.data(), &hp_, dev) == 0,
                  tf::errors::Internal("gaccum_plan_create: ", gaccum_last_error()));
    }
    const int64_t need = gaccum_padded_size(plan_);
    OP_REQUIRES(c, n_accum >= need && n_m >= need && n_v >= need,
                tf::errors::InvalidArgument("accum/m/v slabs hold fewer than gaccum_padded_size() = ", need, " elements"));
    gaccum_step_args a{};
    a.global_step = step;                      // pre-increment value: the Python side feeds one identity() of the counter
    a.accum_n = accum_n_;
    a.lr = lr;
    a.beta1_power = bp(0);
    a.beta2_power = bp(1);
    // TF's compute stream for this device: the kernel is stream-ordered after the backward pass
    // that produced `grads` and before whatever reads the variables next.
    auto* stream = c->op_device_context()->stream();
    gaccum_stream_t cu_stream = stream->platform_specific_handle().stream;   // CUstream
    const int rc = gaccum_step(plan_, grads.data(), params.data(), accum, m, v, &a, cu_stream);
    OP_REQUIRES(c, rc == 0, tf::errors::Internal("gaccum_step: ", gaccum_last_error()));
  }

 private:
  int n_ = 0, accum_n_ = 1;
  gaccum_hparams hp_{};
  std::vector<bool> decay_;
  gaccum_plan* plan_ = nullptr;
};

}  // namespace

REGISTER_KERNEL_BUILDER(
    Name("GaccumStep").Device(tf::DEVICE_GPU).HostMemory("global_step").HostMemory("lr").HostMemory("beta_powers"),
    GaccumStepOpT<false>);
REGISTER_KERNEL_BUILDER(Name("GaccumStepV2")
                            .Device(tf::DEVICE_GPU)
                            .HostMemory("params")
                            .HostMemory("accum")
                            .HostMemory("m")
                            .HostMemory("v")
                            .HostMemory("global_step")
                            .HostMemory("lr")
                            .HostMemory("beta_powers"),
                        GaccumStepOpT<true>);
