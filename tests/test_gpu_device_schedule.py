"""The device schedule on the GPU (include/gaccum.h, gaccum_plan_set_device_schedule).

A device-scheduled train op keeps global_step, the learning rate and the beta powers on the device.  Here it is held,
bit for bit, to the host-scheduled op every other test checks against the oracle:
  - eagerly, over a run that spans the end of warm-up and the end of decay;
  - as ONE captured window (N micro-steps) replayed for the whole run;
  - across checkpoints taken mid-window, host -> device and device -> host;
and a capture that does not start at a window start is refused, on the host and, for a replayed graph that ends
mid-window, by the device.
"""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

MAN = [("bert/embeddings/word_embeddings", (300, 33)), ("bert/embeddings/LayerNorm/gamma", (33,)),
       ("l0/dense/kernel", (64, 64)), ("l0/dense/bias", (64,)), ("big/kernel", (3, 4099))]
N = 3
SCHED = dict(init_lr=1e-3, num_train_steps=12, num_warmup_steps=4)
STEPS = 18                  # past the end of warm-up (4) and of decay (12); a whole number of windows
MULT = [0.5, 1.0, 0.25, 1.0, 2.0]

# (optimizer, clip_norm, dtype, ema, lr multipliers)
CASES = {
    "awd_clip_ema_mult": ("bert", 1.0, torch.float32, True, True),
    "awd_noclip": ("bert", 0.0, torch.float32, False, False),
    "adam": ("adam", 0.0, torch.float32, False, True),
    "adam_clip": ("adam", 1.0, torch.float32, True, False),
    "lamb": ("lamb", 1.0, torch.float32, False, True),
    "bf16_awd": ("bert", 1.0, torch.bfloat16, True, False),
}


def _hp(kind, clip):
    import gaccum_b200 as g
    hp = g.HParams.bert() if kind == "bert" else g.HParams.lamb() if kind == "lamb" else g.HParams.tf_adam()
    hp.clip_norm = clip
    return hp


def _params(dtype):
    rng = np.random.default_rng(11)
    out = []
    for name, shape in MAN:
        a = np.ones(shape, np.float32) if "gamma" in name else rng.normal(0.0, 0.02, size=shape).astype(np.float32)
        out.append(torch.from_numpy(a).cuda().to(dtype))
    return out


def _grads(step, dtype, overflow):
    rng = np.random.Generator(np.random.PCG64(4242 + step))
    gs = [torch.from_numpy(rng.normal(0.0, 0.05, size=s).astype(np.float32)).cuda() for _, s in MAN]
    if overflow and step == 4:          # a loss-scaled window that overflows: skipped on the device
        gs[2][1, 1] = float("inf")
    return [x.to(dtype) for x in gs]


def _op(case, ls, device_schedule, global_step=0):
    import gaccum_b200 as g
    from gaccum_b200 import _lib
    from gaccum_b200.optimization import bert_learning_rate
    from gaccum_b200.train_op import GaccumTrainOp
    kind, clip, dtype, ema, mult = CASES[case]
    kw = {}
    if ls:
        kw["loss_scale"] = _lib.LossScaleConfig(2.0 ** 4, 2.0, 2)
    if ema:
        kw["ema"] = _lib.EmaConfig(0.9, True)
    if mult:
        kw["lr_multipliers"] = MULT
    if device_schedule:
        kw["device_schedule"] = _lib.ScheduleConfig(**SCHED)
        lr_fn = None
    else:
        lr_fn = bert_learning_rate(**SCHED)
    params = _params(dtype)
    return GaccumTrainOp(params, [n for n, _ in MAN], _hp(kind, clip), N, lr_fn, global_step=global_step, **kw), params


def _snapshot(op):
    """Every bit of state the run computes, under the checkpoint's keys (global_step and the beta powers included)."""
    sd = op.state_dict()
    return {k: v.detach().cpu().clone() for k, v in sd.items()}


def _assert_same(a, b, what):
    assert a.keys() == b.keys(), (what, sorted(set(a) ^ set(b)))
    for k in a:
        x, y = a[k], b[k]
        assert x.dtype == y.dtype and x.shape == y.shape, (what, k)
        assert torch.equal(x.view(-1).view(torch.uint8) if x.is_floating_point() else x,
                           y.view(-1).view(torch.uint8) if y.is_floating_point() else y), f"{what}: {k} differs"


def _stats_bits(op):
    st = op.stats()
    return (st["applied"], np.float32(st["lr"]).view(np.uint32), np.float32(st["global_norm"]).view(np.uint32),
            np.float32(st["clip_scale"]).view(np.uint32))


def _eager(op, dtype, overflow, steps=range(STEPS)):
    stats = []
    for s in steps:
        op.run(_grads(s, dtype, overflow))
        stats.append(_stats_bits(op))
    return stats


@pytest.mark.parametrize("ls", [False, True], ids=["nols", "ls"])
@pytest.mark.parametrize("case", sorted(CASES))
def test_device_schedule_matches_host_schedule(case, ls):
    dtype = CASES[case][2]
    host, _ = _op(case, ls, False)
    dev, dparams = _op(case, ls, True)
    assert dev.device_schedule and not host.device_schedule
    s_host = _eager(host, dtype, ls)
    s_dev = _eager(dev, dtype, ls)
    assert s_host == s_dev
    ref = _snapshot(host)
    _assert_same(ref, _snapshot(dev), "eager")
    assert dev.global_step == host.global_step == STEPS
    assert int(dev.global_step_tensor) == STEPS
    if dtype != torch.float32:
        assert all(torch.equal(a, b) for a, b in zip(host.params, dev.params))

    # one captured window replayed for the whole run: reset a device op to step 0 through its checkpoint (after an
    # eager warm-up window that loads every kernel), capture N micro-steps, replay STEPS / N times
    gop, _ = _op(case, ls, True)
    init = gop.state_dict()
    for s in range(N):
        gop.run(_grads(s, dtype, ls))
    gop.load_state_dict(init)
    assert gop.global_step == 0
    static = [[torch.zeros_like(x) for x in _grads(0, dtype, False)] for _ in range(N)]
    graph = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with torch.cuda.graph(graph):
        for i in range(N):
            gop.run(static[i])
    assert gop.global_step == 0                   # nothing ran during the capture
    for w in range(STEPS // N):
        for i in range(N):
            for dst, src in zip(static[i], _grads(w * N + i, dtype, ls)):
                dst.copy_(src)
        graph.replay()
        assert _stats_bits(gop) == s_dev[w * N + N - 1], f"window {w}"
    _assert_same(ref, _snapshot(gop), "graph replay")
    assert gop.global_step == STEPS


@pytest.mark.parametrize("direction", ["host_to_device", "device_to_host"])
@pytest.mark.parametrize("case,ls", [("adam", True), ("lamb", False), ("awd_clip_ema_mult", False),
                                     ("adam_clip", False)])
def test_mid_window_checkpoint_interchanges(case, ls, direction):
    dtype = CASES[case][2]
    ref, _ = _op(case, ls, False)
    s_ref = _eager(ref, dtype, ls)
    cut = 7                                          # mid-window: 7 % N == 1
    first, _ = _op(case, ls, direction == "device_to_host")
    _eager(first, dtype, ls, range(cut))
    sd = first.state_dict()
    assert int(sd["global_step"]) == cut
    second, _ = _op(case, ls, direction == "host_to_device")
    second.load_state_dict(sd)
    assert second.global_step == cut
    s_rest = _eager(second, dtype, ls, range(cut, STEPS))
    assert s_rest == s_ref[cut:]
    _assert_same(_snapshot(ref), _snapshot(second), direction)


def test_capture_that_does_not_start_a_window_is_refused():
    op, _ = _op("adam", False, True)
    op.run(_grads(0, torch.float32, False))            # window position 1 of 3
    graph = torch.cuda.CUDAGraph()
    static = _grads(1, torch.float32, False)
    with pytest.raises(ValueError, match="must start at a window start"):
        with torch.cuda.graph(graph):
            op.run(static)
    # the refused capture launched nothing: the op continues where it was
    assert op.global_step == 1


def test_replayed_graph_that_ends_mid_window_is_refused_on_the_device():
    op, _ = _op("adam", False, True)
    for s in range(N):                                  # warm-up window
        op.run(_grads(s, torch.float32, False))
    static = [_grads(N + i, torch.float32, False) for i in range(2)]
    graph = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with torch.cuda.graph(graph):
        for i in range(2):                              # 2 micro-steps of a 3-step window
            op.run(static[i])
    graph.replay()                                      # steps 3 (apply) and 4: what the schedule selects
    assert op.global_step == N + 2
    before = _snapshot(op)
    graph.replay()                                      # starts with an apply at step 5, an accumulate step
    with pytest.raises(RuntimeError, match="refused a launch at global_step 5"):
        op.schedule_state()
    # nothing changed: the refused launch and every launch after it were no-ops
    with pytest.raises(RuntimeError):
        op.state_dict()
    for i in range(len(MAN)):
        assert torch.equal(op.params[i].cpu(), before[MAN[i][0]])
        assert torch.equal(op.m_view(i).cpu(), before[MAN[i][0] + "/adam_m"])
        assert torch.equal(op.accum_view(i).cpu(), before[MAN[i][0] + "/accum_grad"])
    # writing the step starts the schedule afresh
    op.global_step = N + 2
    assert op.schedule_state()["global_step"] == N + 2


def test_unsupported_combinations_raise():
    from gaccum_b200 import _lib
    from gaccum_b200.train_op import GaccumTrainOp, HostTrainOp
    op, _ = _op("adam", False, True)
    with pytest.raises(ValueError, match="device schedule"):
        op.apply_only()
    with pytest.raises(ValueError, match="device schedule"):
        op.accumulate_only(_grads(0, torch.float32, False))
    with pytest.raises(ValueError, match="pass lr_fn=None"):
        GaccumTrainOp(_params(torch.float32), [n for n, _ in MAN], _hp("adam", 0.0), N, lambda s: 1e-3,
                      device_schedule=_lib.ScheduleConfig(**SCHED))
    host, _ = _op("adam", False, False)
    with pytest.raises(ValueError, match="host"):
        host.global_step_tensor
    with pytest.raises(ValueError, match="device schedule"):
        HostTrainOp([torch.zeros(4)], ["w"], _hp("adam", 0.0), N, lambda s: 1e-3,
                    device_schedule=_lib.ScheduleConfig(**SCHED))


def test_packed_train_op_device_schedule_matches_host():
    import gaccum_b200 as g
    from gaccum_b200 import _lib
    from gaccum_b200.optimization import bert_learning_rate
    from gaccum_b200.train_op import PackedTrainOp
    ops = []
    for dev in (False, True):
        params = _params(torch.float32)
        kw = {"device_schedule": _lib.ScheduleConfig(**SCHED)} if dev else {}
        ops.append(PackedTrainOp(params, [n for n, _ in MAN], _hp("adam", 0.0), N,
                                 None if dev else bert_learning_rate(**SCHED), **kw))
    for op in ops:
        for s in range(STEPS):
            with torch.no_grad():
                for p, gr in zip(op.params, _grads(s, torch.float32, False)):
                    p.grad.add_(gr)
            op.step()
    _assert_same(_snapshot_packed(ops[0]), _snapshot_packed(ops[1]), "packed")
    assert ops[1].global_step == STEPS
    assert ops[1].launches == STEPS and ops[0].launches == STEPS // N


def _snapshot_packed(op):
    out = {"param_slab": op.param_slab.cpu(), "accum": op.accum.cpu(), "m": op.m.cpu(), "v": op.v.cpu()}
    b1, b2 = (op.beta1_power, op.beta2_power) if not op.device_schedule else \
        (op.schedule_state()["beta1_power"], op.schedule_state()["beta2_power"])
    out["beta1_power"] = torch.tensor(b1, dtype=torch.float32)
    out["beta2_power"] = torch.tensor(b2, dtype=torch.float32)
    return out
