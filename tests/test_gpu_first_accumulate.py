"""The first accumulate of a window stores a = +0 + G without reading the accumulators (gaccum.h, gaccum_step).

The accumulators after it are compared with the CPU oracle bit for bit (sign of zero included; any NaN matches any
NaN, since the GPU's add returns the canonical NaN where numpy keeps the payload), and with what the reading kernel
(gaccum_accumulate: a += G) computes from a zeroed accumulator, bit for bit including NaN payloads."""
import numpy as np
import pytest

import oracle_np as onp
from common import make_params, oracle_for

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

# sizes with < 4-element tails, a multi-tile tensor with a tail, an exact tile, a single element, and a tensor that
# never gets a gradient
MAN = [("a/kernel", (777,)), ("a/bias", (5,)), ("b/kernel", (3, 1367)), ("c/kernel", (2048,)), ("one", (1,)),
       ("LayerNorm/gamma", (33,)), ("nograd/kernel", (130,))]
NOGRAD = 6
N = 4
LR = 1e-3


def _bits(x):
    return np.ascontiguousarray(x, np.float32).view(np.uint32)


def _assert_same_bits(got, exp, what):
    got, exp = np.asarray(got, np.float32).ravel(), np.asarray(exp, np.float32).ravel()
    nan = np.isnan(exp)
    assert np.array_equal(np.isnan(got), nan), f"{what}: NaN positions differ"
    bad = np.flatnonzero(_bits(got)[~nan] != _bits(exp)[~nan])
    assert bad.size == 0, f"{what}: {bad.size} elements differ, first {got[~nan][bad[0]]!r} vs {exp[~nan][bad[0]]!r}"


def _special_grads(step, rng):
    """Normal gradients with -0.0, +0.0, NaNs (two payloads), +-inf and subnormals planted in the vector body and in
    the tails; the last tensor has no gradient."""
    specials = np.array([-0.0, 0.0, np.nan, np.inf, -np.inf, 1e-40, -1e-40, 1.4e-45, -1.4e-45],
                        np.float32)
    specials = np.concatenate([specials, np.array([0x7fc12345, 0xffc00001], np.uint32).view(np.float32)])
    out = []
    for i, (_, shape) in enumerate(MAN):
        if i == NOGRAD:
            out.append(None)
            continue
        g = rng.normal(0.0, 0.3, size=shape).astype(np.float32).ravel()
        k = min(g.size, specials.size)
        g[:k] = np.roll(specials, step)[:k]                       # head: vector path (or scalar path if unaligned)
        if g.size > 2 * specials.size:
            g[-k:] = np.roll(specials, step + 3)[:k]              # tail elements included
            g[g.size // 2:g.size // 2 + k] = specials[:k]
        out.append(g.reshape(shape))
    return out


def _device_grads(grads, aligned, flat):
    """Each gradient as its own (256-byte aligned) tensor, or as views into one buffer at odd element offsets
    (4-byte aligned only: the kernel's scalar path)."""
    if aligned:
        return [None if x is None else torch.from_numpy(x).cuda() for x in grads]
    out, o = [], 1
    for x in grads:
        if x is None:
            out.append(None)
            continue
        t = flat[o:o + x.size]
        t.copy_(torch.from_numpy(x.ravel()))
        out.append(t.view(x.shape))
        o = (o + x.size + 3) // 4 * 4 + 1                        # every view starts 4 bytes past a 16-byte boundary
    return out


def _op(params, global_step=0):
    import gaccum_b200 as g
    from gaccum_b200.train_op import GaccumTrainOp
    tp = [torch.from_numpy(p.copy()).cuda() for p in params]
    return GaccumTrainOp(tp, [n for n, _ in MAN], g.HParams.bert(), N, lambda s: LR, global_step=global_step)


@pytest.mark.parametrize("aligned", [True, False], ids=["aligned", "unaligned"])
@pytest.mark.parametrize("window", [1, 2], ids=["after_initial_apply", "later_window"])
def test_first_accumulate_of_window_matches_oracle_bitwise(window, aligned):
    rng = np.random.default_rng(41)
    params = make_params(MAN, rng)
    ref = oracle_for(MAN, params, onp.HParams.bert(), N, constant_lr=LR)
    op = _op(params)
    flat = torch.zeros(sum(int(np.prod(s)) for _, s in MAN) + 8 * len(MAN), device="cuda")
    first = 1 + (window - 1) * N                                 # g - 1 applied, g does not
    for step in range(first + 2):                                # through the first and second accumulate of the window
        grads = _special_grads(step, rng)
        with np.errstate(invalid="ignore", over="ignore"):      # the apply steps see the planted NaNs and infs
            info = ref.run(grads)
        dg = _device_grads(grads, aligned, flat)
        assert op.run(dg) == info.applied
        torch.cuda.synchronize()
        for i in range(len(MAN)):
            _assert_same_bits(op.accum_view(i).cpu().numpy(), ref.accum[i], f"step {step} tensor {i} accum")
        if step == first:
            # the same gradients through the kernel that reads a, onto a zeroed accumulator
            twin = _op(params, global_step=first)
            twin.accumulate_only(dg)
            torch.cuda.synchronize()
            assert torch.equal(op.accum.view(torch.int32), twin.accum.view(torch.int32))
            assert not bool(op.accum_view(NOGRAD).view(torch.int32).any())   # no gradient: left at +0.0
    pad = torch.ones_like(op.accum, dtype=torch.bool)
    for i, (_, s) in enumerate(MAN):
        pad[op.plan.offsets[i]:op.plan.offsets[i] + int(np.prod(s))] = False
    assert not bool(op.accum[pad].view(torch.int32).any())         # padding is never written


def test_packed_first_accumulate_matches_oracle_bitwise():
    """gaccum_step_packed (no pointer table) at the window start g = N + 1, gradients in slab layout."""
    import gaccum_b200 as g
    rng = np.random.default_rng(5)
    params = make_params(MAN, rng)
    plan = g.Plan([int(np.prod(s)) for _, s in MAN], None, g.HParams.bert(), device=0)
    n = plan.padded_size
    pslab, gslab, acc, m, v = (torch.zeros(n, device="cuda") for _ in range(5))
    acc_ref = [np.zeros(s, np.float32) for _, s in MAN]
    grads = _special_grads(0, rng)
    grads[NOGRAD] = np.zeros(MAN[NOGRAD][1], np.float32)           # a slab has no "missing" tensor: zeros
    for x, o, a in zip(grads, plan.offsets, acc_ref):
        gslab[o:o + x.size] = torch.from_numpy(x.ravel())
        np.add(a, x, out=a, dtype=np.float32)
    plan.step_packed(gslab.data_ptr(), pslab.data_ptr(), acc.data_ptr(), m.data_ptr(), v.data_ptr(),
                     g.StepArgs(N + 1, N, 0, LR, 0.9, 0.999, 0.0), -1, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    for i, (o, a) in enumerate(zip(plan.offsets, acc_ref)):
        _assert_same_bits(acc[o:o + a.size].cpu().numpy(), a, f"tensor {i} accum")


def test_accumulate_without_step_arguments_adds_onto_nonzero_accumulator():
    """gaccum_accumulate (accumulate_only) and a forced accumulate branch of gaccum_step_packed read the accumulators
    whatever the step: the data-parallel driver calls the former on the apply step with a non-zero accumulator."""
    import gaccum_b200 as g
    rng = np.random.default_rng(9)
    params = make_params(MAN, rng)
    op = _op(params, global_step=1)                              # a window start: gaccum_step would not read accum
    start = rng.normal(0.0, 1.0, size=op.accum.numel()).astype(np.float32)
    op.accum.copy_(torch.from_numpy(start))
    grads = _special_grads(1, rng)
    op.accumulate_only([None if x is None else torch.from_numpy(x).cuda() for x in grads])
    torch.cuda.synchronize()
    for i, x in enumerate(grads):
        o, sz = op.plan.offsets[i], int(np.prod(MAN[i][1]))
        exp = start[o:o + sz].copy()
        if x is not None:
            np.add(exp, x.ravel(), out=exp, dtype=np.float32)
        _assert_same_bits(op.accum_view(i).cpu().numpy(), exp, f"tensor {i} accum")

    plan = op.plan
    n = plan.padded_size
    gslab, pslab, m, v = (torch.zeros(n, device="cuda") for _ in range(4))
    gvals = rng.normal(0.0, 0.5, size=n).astype(np.float32)
    gslab.copy_(torch.from_numpy(gvals))
    acc = torch.from_numpy(start).cuda()
    plan.step_packed(gslab.data_ptr(), pslab.data_ptr(), acc.data_ptr(), m.data_ptr(), v.data_ptr(),
                     g.StepArgs(1, N, 0, LR, 0.9, 0.999, 0.0), 0, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    got = acc.cpu().numpy()
    for i, (o, (_, s)) in enumerate(zip(plan.offsets, MAN)):
        sz = int(np.prod(s))
        _assert_same_bits(got[o:o + sz], np.add(start[o:o + sz], gvals[o:o + sz], dtype=np.float32),
                          f"forced accumulate, tensor {i}")


def test_window_start_selects_the_kernel_that_does_not_read_accum():
    """Which kernel the step arguments select: at a window start the accumulators are written, not read (a slab
    holding something else than +0.0 there breaks gaccum_step's precondition, and is overwritten with +0 + G); on the
    other accumulate steps they are read.  Steps at and past 2^31 use the reference's int32 cast of global_step."""
    rng = np.random.default_rng(13)
    params = make_params(MAN, rng)
    grads = [None if x is None else torch.from_numpy(x).cuda()
             for x in [rng.normal(0.0, 0.3, size=s).astype(np.float32) if i != NOGRAD else None
                       for i, (_, s) in enumerate(MAN)]]
    for gs, reads in ((1, False), (N + 1, False), (2, True), (N - 1, True), (2**31 + 1, False), (2**31 + 2, True)):
        op = _op(params, global_step=gs)
        op.accum.fill_(7.0)
        assert not op.run(grads)
        torch.cuda.synchronize()
        for i, x in enumerate(grads):
            exp = torch.full_like(op.accum_view(i), 7.0) if x is None else (x + 7.0 if reads else x + 0.0)
            assert torch.equal(op.accum_view(i).view(torch.int32), exp.view(torch.int32)), (gs, i)
