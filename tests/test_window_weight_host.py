"""Per-window normalisation by the window's total weight without a GPU: the C setter's checks on layout-only plans, its
combination with the other setters, the refusals of the entry points that do not support it (C and Python), the byte
counts, the checkpoint key and its TF-format round trip, and the oracle's known answers (W = N is the unweighted oracle;
k-scaled gradients with W = k*N, k a power of two, are too)."""
import ctypes as C
import itertools

import numpy as np
import pytest

import oracle_np as onp
from apply_matrix import reference_op

F32 = np.float32
BLOCK = 0x50000       # a 16-byte aligned address: the setter is host-only and never dereferences it


def _L():
    from gaccum_b200 import _lib
    return _lib, _lib._load()


def _plan(variant=0):
    import gaccum_b200 as g
    hp = g.HParams(variant, 0, 0.9, 0.999, 1e-6, 0.01, 1.0)
    return g.Plan([1000, 37, 5], [True, False, True], hp, device=-1)


def _set(plan, addr):
    lib, L = _L()
    return L.gaccum_plan_set_window_weight(plan._h, addr)


# ---- the C ABI on layout-only plans --------------------------------------------------------------------------------
@pytest.mark.parametrize("bad", [None, BLOCK + 4, BLOCK + 8, BLOCK + 1])
def test_setter_refuses_null_and_misaligned_blocks(bad):
    lib, L = _L()
    assert _set(_plan(), bad) == lib.EINVAL
    assert "16-byte aligned" in L.gaccum_last_error().decode()


def test_setter_refuses_a_null_plan():
    lib, L = _L()
    assert L.gaccum_plan_set_window_weight(None, BLOCK) == lib.EINVAL


@pytest.mark.parametrize("variant", [0, 1, 2])
def test_setter_accepts_an_aligned_block(variant):
    plan = _plan(variant)
    assert _set(plan, BLOCK) == 0
    assert _set(plan, BLOCK + 16) == 0                                     # may be called again before compute


def test_setter_is_refused_after_a_compute_call():
    lib, L = _L()
    plan = _plan()
    args = lib.StepArgs(0, 1, 0, 1e-3, 0.9, 0.999, 0.0)
    assert L.gaccum_apply(plan._h, None, None, None, None, None, C.byref(args), None) != 0   # counts as a compute call
    assert _set(plan, BLOCK) == lib.EINVAL
    assert "before the plan's first compute call" in L.gaccum_last_error().decode()


@pytest.mark.parametrize("order", list(itertools.permutations(["ww", "lr_mult", "ema", "dtype", "loss_scale", "adapt"])))
def test_setters_combine_in_any_order(order):
    lib, L = _L()
    plan = _plan(variant=2)
    calls = {
        "ww": lambda: _set(plan, BLOCK),
        "lr_mult": lambda: L.gaccum_plan_set_lr_multipliers(plan._h, C.cast((C.c_float * 3)(0.5, 0.0, 2.0), C.c_void_p)),
        "ema": lambda: L.gaccum_plan_set_ema(plan._h, C.byref(lib.EmaConfig(0.999)), 0x10000, 0x20000),
        "dtype": lambda: L.gaccum_plan_set_param_dtype(plan._h, lib.DTYPE_BF16, 0x30000),
        "loss_scale": lambda: L.gaccum_plan_set_loss_scale(plan._h, C.byref(lib.LossScaleConfig()), 0x40000),
        "adapt": lambda: L.gaccum_plan_set_layer_adaptation(plan._h, C.cast((C.c_uint8 * 3)(1, 0, 1), C.c_void_p)),
    }
    for what in order:
        assert calls[what]() == 0, what
    assert plan.algorithmic_bytes(True) == 56 * plan.num_elements


@pytest.mark.parametrize("variant, apply_bytes", [(0, 36), (1, 36), (2, 48)])
def test_algorithmic_bytes_unchanged(variant, apply_bytes):
    plan = _plan(variant)
    acc = plan.algorithmic_bytes(False)
    assert _set(plan, BLOCK) == 0
    assert plan.algorithmic_bytes(True) == apply_bytes * plan.num_elements
    assert plan.algorithmic_bytes(False) == acc


def test_data_parallel_and_host_session_refuse_a_weighted_plan():
    lib, L = _L()
    plan = _plan()
    assert _set(plan, BLOCK) == 0
    comm = lib.DpComm()
    comm.world = 2
    args = lib.StepArgs(0, 1, 0, 1e-3, 0.9, 0.999, 0.0)
    for fn in (L.gaccum_step_dp, L.gaccum_apply_dp):
        assert fn(plan._h, C.byref(comm), None, None, None, C.byref(args), 1, None) == lib.EINVAL
        assert "window weight" in L.gaccum_last_error().decode()
    h = C.c_void_p()
    assert L.gaccum_host_session_create(C.byref(h), plan._h) == lib.EINVAL
    assert "window weight" in L.gaccum_last_error().decode()


# ---- Python ----------------------------------------------------------------------------------------------------------
def test_python_front_ends_refuse_a_window_weight():
    import torch
    import gaccum_b200 as g
    from gaccum_b200.distributed import FusedDataParallelTrainOp
    from gaccum_b200.train_op import HostTrainOp
    with pytest.raises(ValueError, match="window weight"):
        HostTrainOp([torch.zeros(4)], ["w"], g.HParams.bert(), 2, lambda s: 1e-3, window_weight=True)
    with pytest.raises(ValueError, match="window weight"):
        FusedDataParallelTrainOp([torch.zeros(4)], ["w"], g.HParams.bert(), 2, lambda s: 1e-3, window_weight=True)


def test_checkpoint_key_maps_both_ways_as_an_fp32_scalar():
    import torch
    from gaccum_b200 import tf_checkpoint as tfc
    from gaccum_b200.train_op import WINDOW_WEIGHT_KEY
    assert WINDOW_WEIGHT_KEY == "gradient_accumulation/window_weight"
    names = ["w/kernel"]
    sd = {"global_step": torch.tensor(5), "w/kernel": torch.ones(3), "w/kernel/adam_m": torch.zeros(3),
          "w/kernel/adam_v": torch.zeros(3), "w/kernel/accum_grad": torch.zeros(3),
          WINDOW_WEIGHT_KEY: torch.tensor(1040.0)}
    ref = tfc.to_reference_names(sd, names, 0)
    assert ref[WINDOW_WEIGHT_KEY].dtype == np.float32 and ref[WINDOW_WEIGHT_KEY].shape == () and ref[WINDOW_WEIGHT_KEY] == 1040
    back = tfc.from_reference_names(ref, names, 0, window_weight=True)
    assert back[WINDOW_WEIGHT_KEY].dtype == np.float32 and float(back[WINDOW_WEIGHT_KEY]) == 1040.0
    del ref[WINDOW_WEIGHT_KEY]
    with pytest.raises(KeyError, match="window_weight"):
        tfc.from_reference_names(ref, names, 0, window_weight=True)
    assert WINDOW_WEIGHT_KEY not in tfc.from_reference_names(ref, names, 0)          # an unweighted op needs none


# ---- the oracle ------------------------------------------------------------------------------------------------------
MAN = [("a/kernel", (300,)), ("a/bias", (7,)), ("LayerNorm/gamma", (5,)), ("b/kernel", (4, 9))]
MODES = ["noclip", "clip", "ls_noclip", "ls_clip"]
VARIANTS = ["adamw", "adam", "lamb"]


def _same(a, b, k=1.0):
    for xs, ys in ((a.params, b.params), (a.m, b.m), (a.v, b.v)):
        for x, y in zip(xs, ys):
            assert x.tobytes() == y.tobytes()
    with np.errstate(over="ignore", invalid="ignore"):
        for x, y in zip(a.accum, b.accum):                 # the weighted run accumulates k-scaled gradients, exactly
            assert x.tobytes() == np.multiply(y, F32(k), dtype=F32).tobytes()
    assert F32(a.scale).tobytes() == F32(b.scale).tobytes()
    assert [F32(r).tobytes() for r in a.ratios] == [F32(r).tobytes() for r in b.ratios]


@pytest.mark.parametrize("k", [1.0, 4.0, 0.25])
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("variant", VARIANTS)
def test_oracle_with_w_equal_k_n_and_k_scaled_gradients_is_unweighted(variant, mode, k):
    N = 3
    rng = np.random.default_rng(0)
    params = [rng.normal(0, 0.05, s).astype(F32) for _, s in MAN]
    w = reference_op(variant, mode, params, [n for n, _ in MAN], N, window_weight=True)
    u = reference_op(variant, mode, params, [n for n, _ in MAN], N)
    for s in range(10):
        grads = [rng.normal(0, 0.1, sh).astype(F32) for _, sh in MAN]
        if mode.startswith("ls_") and s == 4:
            grads[0][3] = np.inf
        S = F32(u.scale)
        with np.errstate(over="ignore", invalid="ignore"):
            gu = [g * S for g in grads]
            gw = [g * S * F32(k) for g in grads]
        iw = w.run(gw, weight=k * (N if s == 0 else 1))
        iu = u.run(gu)
        assert iw.applied == iu.applied
        _same(w, u, k)
    assert w.last_weight == F32(k * N) and w.weight == 0


def test_oracle_divides_by_the_weight():
    rng = np.random.default_rng(1)
    params = [rng.normal(0, 0.05, s).astype(F32) for _, s in MAN]
    w = reference_op("adamw", "noclip", params, [n for n, _ in MAN], 2, window_weight=True)
    w.global_step = 1
    g1 = [rng.normal(0, 0.1, sh).astype(F32) for _, sh in MAN]
    g2 = [rng.normal(0, 0.1, sh).astype(F32) for _, sh in MAN]
    w.run(g1, weight=3.0)
    m_before = [m.copy() for m in w.m]
    w.run(g2, weight=37.0)
    c = [np.divide(np.add(a, b, dtype=F32), F32(40.0), dtype=F32) for a, b in zip(g1, g2)]
    omb1 = F32(1.0 - 0.9)
    for m0, m1, ci in zip(m_before, w.m, c):
        assert np.array_equal(m1, np.add(np.multiply(F32(0.9), m0, dtype=F32), np.multiply(omb1, ci, dtype=F32), dtype=F32))
    assert w.last_weight == 40.0 and w.weight == 0.0


def test_unweighted_oracle_refuses_a_weight():
    params = [np.zeros(s, F32) for _, s in MAN]
    u = reference_op("adamw", "noclip", params, [n for n, _ in MAN], 2)
    with pytest.raises(ValueError, match="window weight"):
        u.run([None] * len(MAN), weight=1.0)
    assert u.global_step == 0


# ---- the data-parallel driver at world 2 over gloo ------------------------------------------------------------------
DP_MAN = [("l0/kernel", (33, 7)), ("l0/bias", (7,)), ("LayerNorm/gamma", (7,)), ("emb", (301,))]
DP_N, DP_STEPS, DP_WORLD, DP_CUT = 3, 8, 2, 5


class WeightedOracleEngine:
    """Test-only adapter: a weighted ``ComposedReferenceTrainOp`` behind the engine interface ``DataParallelTrainOp`` drives
    (GaccumTrainOp's), its accumulators aliased to one flat slab and its running W in a 0-dim fp32 tensor,
    ``window_weight``, as a weighted GaccumTrainOp exposes it."""

    def __init__(self, ref):
        import torch
        self.ref = ref
        flat = np.zeros(sum(a.size for a in ref.accum), F32)
        o = 0
        for i, a in enumerate(ref.accum):
            ref.accum[i] = flat[o:o + a.size].reshape(a.shape); o += a.size
        self.accum = torch.from_numpy(flat)
        self.window_weight = torch.zeros((), dtype=torch.float32)
        self.N = ref.N

    @property
    def global_step(self):
        return self.ref.global_step

    @global_step.setter
    def global_step(self, v):
        self.ref.global_step = v

    def _add_weight(self, weight):
        if weight is None:
            raise ValueError("every micro-step needs its weight")
        self.window_weight.add_(float(F32(weight)))

    def _run_ref(self, grads):
        self.ref.weight = F32(self.window_weight.item())
        info = self.ref.run(grads)
        self.window_weight.fill_(float(self.ref.weight))
        return info

    def run(self, grads, weight=None):
        self._add_weight(weight)
        return self._run_ref(grads).applied

    def accumulate_only(self, grads):
        for a, g in zip(self.ref.accum, grads):
            if g is not None:
                np.add(a, g, out=a)

    def apply_only(self, grads):
        assert grads is None and self.ref.global_step % self.N == 0
        self._run_ref([None] * len(self.ref.accum))

    def state_dict(self):
        import torch
        from gaccum_b200.train_op import WINDOW_WEIGHT_KEY
        out = {"global_step": torch.tensor(self.ref.global_step), WINDOW_WEIGHT_KEY: self.window_weight.clone()}
        flat = self.accum.numpy()
        o = 0
        for i, n in enumerate(self.ref.names):
            sz = self.ref.params[i].size
            out[n] = torch.from_numpy(self.ref.params[i].copy())
            out[n + "/adam_m"] = torch.from_numpy(self.ref.m[i].copy())
            out[n + "/adam_v"] = torch.from_numpy(self.ref.v[i].copy())
            out[n + "/accum_grad"] = torch.from_numpy(flat[o:o + sz].reshape(self.ref.params[i].shape).copy())
            o += sz
        return out

    def load_state_dict(self, sd, strict=True):
        from gaccum_b200.train_op import WINDOW_WEIGHT_KEY
        self.ref.global_step = int(sd["global_step"])
        self.window_weight.fill_(float(sd[WINDOW_WEIGHT_KEY]))
        for i, n in enumerate(self.ref.names):
            self.ref.params[i][...] = sd[n].numpy(); self.ref.m[i][...] = sd[n + "/adam_m"].numpy()
            self.ref.v[i][...] = sd[n + "/adam_v"].numpy(); self.ref.accum[i][...] = sd[n + "/accum_grad"].numpy()


def _dp_grads(rank, step):
    """This rank's gradient of its SUMMED loss (a weighted producer does not divide by num_workers) and its weight."""
    rng = np.random.Generator(np.random.PCG64(4242 + 1000 * rank + step))
    return [rng.normal(0, 0.3, s).astype(F32) for _, s in DP_MAN], float(rng.integers(1, 60))


def _dp_ref(fill=None):
    rng = np.random.default_rng(5)
    params = [rng.normal(0, 0.02, s).astype(F32) if fill is None else np.full(s, fill, F32) for _, s in DP_MAN]
    return reference_op("adamw", "clip", params, [n for n, _ in DP_MAN], DP_N, window_weight=True)


def _dp_worker(rank, port, outdir):
    import os
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for p in (root, os.path.join(root, "oracle"), os.path.join(root, "tests")):
        sys.path.insert(0, p)
    import torch.distributed as dist
    from gaccum_b200.distributed import DataParallelTrainOp
    from gaccum_b200.train_op import WINDOW_WEIGHT_KEY
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=DP_WORLD)
    ref = _dp_ref()
    dp = DataParallelTrainOp(WeightedOracleEngine(ref), None)
    last = []
    for s in range(DP_CUT):                               # N = 3: steps 0 and 3 apply, step 4 leaves a window open
        g, w = _dp_grads(rank, s)
        dp.run(g, weight=w)
        last.append(float(ref.last_weight))
    local_w = float(dp.engine.window_weight)
    sd = dp.state_dict()                                  # collective: accumulators and W summed over ranks
    ref2 = _dp_ref(fill=9.0)                              # a restarted worker holds garbage until it loads
    dp2 = DataParallelTrainOp(WeightedOracleEngine(ref2), None)
    dp2.load_state_dict(sd)
    w_after_load = float(dp2.engine.window_weight)
    for s in range(DP_CUT, DP_STEPS):
        g, w = _dp_grads(rank, s)
        dp2.run(g, weight=w)
        last.append(float(ref2.last_weight))
    np.savez(os.path.join(outdir, f"rank{rank}.npz"), *ref2.params, *ref2.m, *ref2.v, local_w=local_w,
             sd_w=float(sd[WINDOW_WEIGHT_KEY]), w_after_load=w_after_load, last=np.array(last),
             allreduces=dp.allreduces + dp2.allreduces, w_end=float(dp2.engine.window_weight))
    dist.destroy_process_group()


def test_data_parallel_driver_sums_the_window_weight_over_ranks(tmp_path):
    import socket
    import torch.multiprocessing as mp
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]
    mp.spawn(_dp_worker, args=(port, str(tmp_path)), nprocs=DP_WORLD, join=True)
    r0, r1 = np.load(tmp_path / "rank0.npz"), np.load(tmp_path / "rank1.npz")
    T = len(DP_MAN)
    w = [[_dp_grads(r, s)[1] for s in range(DP_STEPS)] for r in range(DP_WORLD)]
    # mid-window state_dict: the open window's W (step 4) summed over ranks; rank 0 resumes with it, rank 1 from zero
    assert float(r0["local_w"]) == w[0][4] and float(r1["local_w"]) == w[1][4]
    assert float(r0["sd_w"]) == float(r1["sd_w"]) == w[0][4] + w[1][4]
    assert float(r0["w_after_load"]) == w[0][4] + w[1][4] and float(r1["w_after_load"]) == 0.0
    # every apply divided by the global window's total: W of step 0, steps 1-3, steps 4-6
    totals = [w[0][0] + w[1][0], sum(w[0][1:4]) + sum(w[1][1:4]), sum(w[0][4:7]) + sum(w[1][4:7])]
    for rank, r in enumerate((r0, r1)):
        last = list(r["last"])
        assert last[0] == totals[0] and last[3] == totals[1] and last[6] == totals[2], last
        assert float(r["w_end"]) == w[rank][7]            # between applies W stays rank-local
        assert int(r["allreduces"]) == 3                  # one exchange per window
    for i in range(3 * T):                                # replicas are identical
        assert np.array_equal(r0[f"arr_{i}"], r1[f"arr_{i}"]), i
    # a single process fed the rank-summed gradients and weights
    ref = _dp_ref()
    for s in range(DP_STEPS):
        (g0, w0), (g1, w1) = _dp_grads(0, s), _dp_grads(1, s)
        ref.run([a + b for a, b in zip(g0, g1)], weight=w0 + w1)
    for i in range(T):
        np.testing.assert_allclose(r0[f"arr_{i}"], ref.params[i], rtol=1e-5, atol=1e-7)
        np.testing.assert_allclose(r0[f"arr_{T + i}"], ref.m[i], rtol=1e-5, atol=1e-7)
        np.testing.assert_allclose(r0[f"arr_{2 * T + i}"], ref.v[i], rtol=1e-5, atol=1e-9)
    # the per-token mean differs from the mean of the ranks' means: the weights matter
    unweighted = _dp_ref()
    for s in range(DP_STEPS):
        (g0, w0), (g1, w1) = _dp_grads(0, s), _dp_grads(1, s)
        unweighted.run([a + b for a, b in zip(g0, g1)], weight=DP_N * 2 if s == 0 else 2.0)
    assert not np.allclose(r0["arr_0"], unweighted.params[0], rtol=1e-5, atol=1e-7)
