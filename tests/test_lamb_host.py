"""LAMB without a GPU: the oracle's known answers and its agreement with an fp64 closed form written from the paper,
the C ABI's setter / readback checks and refusals, the algorithmic bytes, the checkpoint names and the TF adapter's
refusal of variant 2."""
import ctypes as C
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

import oracle_np as onp
from composed_oracle import ComposedReferenceTrainOp, lamb_update, norm

F32 = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _hp(**kw):
    return onp.HParams(variant=2, **kw)


# ---- oracle known answers ------------------------------------------------------------------------------------------
def test_one_element_adapted_tensor_moves_by_lr_times_p():
    for p0, g in ((0.75, 0.3), (-2.5, 1e-3), (1e-3, -7.0)):
        p, m, v = (np.array([x], F32) for x in (p0, 0.0, 0.0))
        p2, _, _, r = lamb_update(p, m, v, np.array([g], F32), 0.125, 0.9, 0.999, 1e-6, 0.0, False, True, 0.9, 0.999)
        assert abs(abs(float(p2[0] - p[0])) - 0.125 * abs(p0)) <= 1e-6 * 0.125 * abs(p0)


def test_zero_weights_or_zero_update_give_ratio_one():
    z = np.zeros(5, F32)
    c = np.full(5, 0.5, F32)
    # p = 0: r = 1, the step is the plain bias-corrected update
    p2, _, _, r = lamb_update(z.copy(), z.copy(), z.copy(), c, 0.1, 0.9, 0.999, 1e-6, 0.0, False, True, 0.9, 0.999)
    assert r == 1.0 and np.all(p2 < 0)
    # u = 0 (zero gradient, no decay): r = 1 and p unchanged
    p = np.arange(5, dtype=F32)
    p2, _, _, r = lamb_update(p.copy(), z.copy(), z.copy(), z, 0.1, 0.9, 0.999, 1e-6, 0.0, False, True, 0.9, 0.999)
    assert r == 1.0 and np.array_equal(p2, p)


def test_without_adaptation_the_update_is_bias_corrected_adamw():
    rng = np.random.default_rng(1)
    p, m, v, c = (rng.normal(0, s, 50).astype(F32) for s in (0.05, 0.01, 0.0, 0.1))
    v = np.abs(v) + F32(1e-4)
    b1p, b2p = F32(0.9) ** 3, F32(0.999) ** 3
    p2, m2, v2, r = lamb_update(p, m, v, c, 1e-3, 0.9, 0.999, 1e-6, 0.01, True, False, b1p, b2p)
    assert r == 1.0
    m64 = 0.9 * m.astype(np.float64) + 0.1 * c
    v64 = 0.999 * v.astype(np.float64) + 0.001 * c.astype(np.float64) ** 2
    u = (m64 / (1 - float(b1p))) / (np.sqrt(v64 / (1 - float(b2p))) + 1e-6) + 0.01 * p
    np.testing.assert_allclose(p2, p - 1e-3 * u, rtol=1e-6, atol=1e-9)


def _closed_form_run(params, names, grads_seq, N, lr, b1, b2, eps, wd, clip, decay, adapt):
    """LAMB (You et al. 2019, Algorithm 2) with gradient accumulation and clipping, all in fp64."""
    p = [x.astype(np.float64) for x in params]
    m = [np.zeros_like(x) for x in p]
    v = [np.zeros_like(x) for x in p]
    acc = [np.zeros_like(x) for x in p]
    t = 0
    for step, grads in enumerate(grads_seq):
        for a, g in zip(acc, grads):
            a += g
        if step % N == 0:
            c = [a / N for a in acc]
            if clip > 0:
                gn = math.sqrt(sum(float(np.sum(x * x)) for x in c))
                c = [x * (clip / max(gn, clip)) for x in c]
            t += 1
            for i in range(len(p)):
                m[i] = b1 * m[i] + (1 - b1) * c[i]
                v[i] = b2 * v[i] + (1 - b2) * c[i] ** 2
                u = (m[i] / (1 - b1 ** t)) / (np.sqrt(v[i] / (1 - b2 ** t)) + eps)
                if decay[i]:
                    u = u + wd * p[i]
                wn, un = np.linalg.norm(p[i]), np.linalg.norm(u)
                r = wn / un if (adapt[i] and wn > 0 and un > 0) else 1.0
                p[i] = p[i] - lr * r * u
            acc = [np.zeros_like(x) for x in p]
    return p


@pytest.mark.parametrize("seed", range(6))
def test_oracle_agrees_with_fp64_closed_form(seed):
    rng = np.random.default_rng(100 + seed)
    man = [("w/kernel", (int(rng.integers(1, 300)),)), ("w/bias", (int(rng.integers(1, 40)),)),
           ("LayerNorm/gamma", (int(rng.integers(1, 40)),)), ("emb", (int(rng.integers(100, 900)),))]
    N = int(rng.integers(1, 5))
    clip = float(rng.choice([0.0, 1.0, 0.05]))
    wd = float(rng.choice([0.0, 0.01, 0.1]))
    names = [n for n, _ in man]
    params = [rng.normal(0, 0.05, s).astype(F32) for _, s in man]
    grads = [[rng.normal(0, 0.1, s).astype(F32) for _, s in man] for _ in range(3 * N + 1)]
    ref = ComposedReferenceTrainOp([x.copy() for x in params], names, _hp(weight_decay_rate=wd, clip_norm=clip), N,
                                   constant_lr=1e-3, adapt_exclude=["LayerNorm"])
    for g in grads:
        ref.run(g)
    exp = _closed_form_run(params, names, grads, N, float(F32(1e-3)), 0.9, 0.999, 1e-6, wd, clip, ref.decay, ref.adapt)
    for got, e, p0 in zip(ref.params, exp, params):
        # the relative error of the step (p - p0), not of p
        step = np.max(np.abs(e - p0.astype(np.float64)))
        assert np.max(np.abs(got.astype(np.float64) - e)) <= 1e-6 * max(np.max(np.abs(e)), 1e-30) + 1e-4 * step


def test_norm_is_fp64_sum_rounded_once():
    x = np.full(1 << 20, 1.0 + 2.0 ** -12, F32)
    assert norm(x) == np.sqrt(F32(np.sum(x.astype(np.float64) ** 2)), dtype=F32)


# ---- the C ABI on layout-only plans --------------------------------------------------------------------------------
def _L():
    from gaccum_b200 import _lib
    return _lib, _lib._load()


def _plan(variant=2):
    import gaccum_b200 as g
    hp = g.HParams.lamb() if variant == 2 else (g.HParams.bert() if variant == 0 else g.HParams.tf_adam())
    return g.Plan([10, 3000, 1], None, hp, device=-1)


def test_set_layer_adaptation_checks():
    _lib, L = _L()
    mask = (C.c_uint8 * 3)(1, 0, 1)
    assert L.gaccum_plan_set_layer_adaptation(None, mask) == _lib.EINVAL
    assert L.gaccum_plan_set_layer_adaptation(_plan()._h, None) == _lib.EINVAL
    for variant in (0, 1):
        assert L.gaccum_plan_set_layer_adaptation(_plan(variant)._h, mask) == _lib.EINVAL
        assert "GACCUM_LAMB" in L.gaccum_last_error().decode()
    plan = _plan()
    assert L.gaccum_plan_set_layer_adaptation(plan._h, mask) == _lib.OK
    with pytest.raises(_lib.GaccumError) as e:                   # a compute call, refused without a device, still counts
        plan.step_packed(0x1000, 0x1000, 0x1000, 0x1000, 0x1000, _lib.StepArgs(0, 1, 0, 1e-3, 0.9, 0.999, 0.0), 1)
    assert e.value.code == _lib.ENODEVICE
    assert L.gaccum_plan_set_layer_adaptation(plan._h, mask) == _lib.EINVAL
    assert "before the plan's first compute call" in L.gaccum_last_error().decode()
    with pytest.raises(ValueError):
        _plan().set_layer_adaptation([True])


def test_read_trust_ratios_checks():
    _lib, L = _L()
    out = (C.c_float * 3)()
    assert L.gaccum_read_trust_ratios(None, out, None) == _lib.EINVAL
    assert L.gaccum_read_trust_ratios(_plan()._h, None, None) == _lib.EINVAL
    assert L.gaccum_read_trust_ratios(_plan(0)._h, out, None) == _lib.EINVAL
    assert L.gaccum_read_trust_ratios(_plan()._h, out, None) == _lib.ENODEVICE


def test_variant_2_is_accepted_and_3_is_not():
    import gaccum_b200 as g
    _lib, _ = _L()
    assert g.LAMB == _lib.LAMB == 2
    with pytest.raises(_lib.GaccumError):
        g.Plan([4], None, g.HParams(3, 0, 0.9, 0.999, 1e-6, 0.0, 0.0), device=-1)


def test_algorithmic_bytes_48_per_param():
    plan = _plan()
    P = 10 + 3000 + 1
    assert plan.algorithmic_bytes(True) == 48 * P and plan.algorithmic_bytes(False) == 12 * P
    assert _plan(0).algorithmic_bytes(True) == 36 * P


def test_data_parallel_and_host_entry_points_refuse_lamb():
    _lib, L = _L()
    plan = _plan()
    args = _lib.StepArgs(0, 1, 0, 1e-3, 0.9, 0.999, 0.0)
    comm = _lib.DpComm()
    comm.world, comm.rank = 2, 0
    for fn in (L.gaccum_step_dp, L.gaccum_apply_dp):
        assert fn(plan._h, C.byref(comm), None, None, None, C.byref(args), 1, None) == _lib.EINVAL
        assert "GACCUM_LAMB" in L.gaccum_last_error().decode()
    h = C.c_void_p()
    assert L.gaccum_host_session_create(C.byref(h), plan._h) == _lib.EINVAL
    assert "GACCUM_LAMB" in L.gaccum_last_error().decode()


def test_python_front_ends_refuse_lamb():
    torch = pytest.importorskip("torch")
    import gaccum_b200 as g
    from gaccum_b200.distributed import FusedDataParallelTrainOp
    from gaccum_b200.train_op import HostTrainOp
    p = [torch.zeros(4)]
    with pytest.raises(ValueError, match="LAMB"):
        FusedDataParallelTrainOp(p, ["w"], g.HParams.lamb(), 2, lambda s: 1e-3)
    with pytest.raises(ValueError, match="LAMB"):
        HostTrainOp(p, ["w"], g.HParams.lamb(), 2, lambda s: 1e-3)


def test_optimizer_classes_and_create_optimizer_attribute():
    from gaccum_b200 import optimization as opt
    assert opt.optimizer_type == "adam"
    o = opt.LAMBOptimizer(1e-3, exclude_from_weight_decay=["bias", "LayerNorm"])
    assert o.exclude_from_layer_adaptation == ["bias", "LayerNorm"]
    assert o._do_use_weight_decay("a/kernel") and not o._do_use_weight_decay("a/bias")
    assert o._do_layer_adaptation("a/kernel:0") and not o._do_layer_adaptation("x/LayerNorm/gamma:0")
    o0 = opt.LAMBOptimizer(1e-3, weight_decay_rate=0.0, exclude_from_weight_decay=["bias"])
    assert not o0._do_use_weight_decay("a/kernel") and o0._do_layer_adaptation("a/kernel")   # by name, whatever wd
    assert not o0._do_layer_adaptation("a/bias")
    o2 = opt.LAMBOptimizer(1e-3, exclude_from_weight_decay=["bias"], exclude_from_layer_adaptation=[])
    assert o2._do_layer_adaptation("a/bias")
    hp = o._hparams(1.0)
    assert (hp.variant, hp.weight_decay_rate, hp.epsilon, hp.clip_norm) == (2, 0.01, 1e-6, 1.0)


def test_tf_checkpoint_names_round_trip_for_variant_2():
    from gaccum_b200 import tf_checkpoint as tc
    names = ["a/kernel", "a/bias"]
    rng = np.random.default_rng(2)
    state = {"global_step": np.int64(7), "beta1_power": F32(0.9 ** 3), "beta2_power": F32(0.999 ** 3)}
    for n, s in zip(names, ((3, 4), (4,))):
        state[n] = rng.normal(size=s).astype(F32)
        for k in ("/adam_m", "/adam_v", "/accum_grad"):
            state[n + k] = rng.normal(size=s).astype(F32)
    ref = tc.to_reference_names(state, names, 2)
    assert {"a/kernel/lamb_m", "a/kernel/lamb_v", "a/bias/lamb_m", "beta1_power", "beta2_power"} <= set(ref)
    back = tc.from_reference_names(ref, names, 2)
    assert set(back) == set(state)
    for k in state:
        assert np.array_equal(np.asarray(back[k]), np.asarray(state[k])), k
    shim = tc.to_shim_names(ref, names, 2)
    assert np.array_equal(shim["gaccum/beta_powers"], np.asarray([state["beta1_power"], state["beta2_power"]], F32))
    again = tc.from_shim_names(shim, names, 2)
    for k in ref:
        assert np.array_equal(np.asarray(again[k]), np.asarray(ref[k])), k


def test_tf_checkpoint_cli_accepts_variant_2(tmp_path):
    from gaccum_b200 import tf_checkpoint as tc
    names = ["w"]
    ref = {"global_step": np.int64(1), "w": np.ones(3, F32), "w/lamb_m": np.zeros(3, F32), "w/lamb_v": np.zeros(3, F32),
           "Variable": np.zeros(3, F32), "beta1_power": F32(0.9), "beta2_power": F32(0.999)}
    tc.write_bundle(str(tmp_path / "in"), ref)
    (tmp_path / "names").write_text("w\n")
    assert tc._main(["convert", "to-shim", str(tmp_path / "in"), str(tmp_path / "out"), "--names",
                     str(tmp_path / "names"), "--variant", "2"]) == 0
    out = tc.read_bundle(str(tmp_path / "out"))
    assert np.allclose(out["gaccum/beta_powers"], [0.9, 0.999])


_DRIVER = r"""
#include <cstdio>
#include <memory>
#include <string>
#include "gaccum.h"
#include "tensorflow/core/framework/op_kernel.h"
namespace tf = tensorflow;
int main() {
  for (const char* op : {"GaccumStep", "GaccumStepV2"}) {
    for (int variant : {0, 1, 2, -1}) {
      tf::OpKernelConstruction c;
      c.attrs["N"].i = 1; c.attrs["accum_n"].i = 2; c.attrs["variant"].i = variant;
      c.attrs["beta1"].s = "0.9"; c.attrs["beta2"].s = "0.999"; c.attrs["epsilon"].s = "1e-06";
      c.attrs["weight_decay_rate"].s = "0.01"; c.attrs["clip_norm"].s = "1.0"; c.attrs["decay_mask"].bl = {true};
      auto& reg = tf::MockRegistry::Get();
      std::unique_ptr<tf::OpKernel> k(reg.kernels.find(op)->second.second(&c));
      std::printf("%s %d %s\n", op, variant, c.status.ok() ? "ok" : c.status.ToString().c_str());
    }
  }
  return 0;
}
"""


def test_tf_adapter_rejects_variant_2(tmp_path):
    """tf_shim/gaccum_tf_op.cc over tests/tf_mock: the op refuses variant 2 (and any other but 0 and 1) with
    InvalidArgument when it is constructed -- LAMB has no trust-ratio state or adaptation mask in the TF graph."""
    import gaccum_b200 as g
    gxx = shutil.which("g++") or shutil.which("c++") or pytest.skip("no g++ in this image")
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    src = tmp_path / "variant_driver.cc"
    src.write_text(_DRIVER)
    lib = g.lib_path()
    out = str(tmp_path / "variant_driver")
    cmd = [gxx, "-std=c++17", "-O1", "-I", os.path.join(ROOT, "tests", "tf_mock"), "-I", os.path.join(ROOT, "include"),
           "-I", os.path.join(cuda, "include"),
           os.path.join(ROOT, "gradient-accumulation-tf-estimator_b200", "tf_shim", "gaccum_tf_op.cc"), str(src), "-o", out,
           lib, "-L", os.path.join(cuda, "lib64"), "-lcudart", "-Wl,-rpath," + os.path.dirname(lib),
           "-Wl,-rpath," + os.path.join(cuda, "lib64")]
    env = dict(os.environ); env.pop("CC", None); env.pop("CXX", None)
    r = subprocess.run(cmd, capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([out], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stderr
    lines = r.stdout.splitlines()
    for op in ("GaccumStep", "GaccumStepV2"):
        assert f"{op} 0 ok" in lines and f"{op} 1 ok" in lines
        for v in (2, -1):
            line = next(l for l in lines if l.startswith(f"{op} {v} "))
            assert "variant must be 0" in line, line          # refused when the op is constructed, not at Compute()
