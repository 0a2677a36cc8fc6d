"""16-bit models without a GPU: the C ABI's gaccum_plan_set_param_dtype argument checks, its refusal after a compute
call (in either order with loss scaling), the algorithmic bytes of a 16-bit plan, the entry points that refuse such a
plan, and the Python train ops that refuse 16-bit parameters."""
import ctypes as C

import pytest

MASTER = 0x1000        # a 16-byte aligned address: the setter validates on the host and never dereferences it
ARGS = (0, 1, 0, 1e-3, 0.9, 0.999, 0.0)


def _lib():
    from gaccum_b200 import _lib
    return _lib


def _plan(numels=(10, 3000)):
    import gaccum_b200 as g
    return g.Plan(list(numels), None, g.HParams.bert(), device=-1)


def _set(plan, dtype, master=MASTER):
    return _lib()._load().gaccum_plan_set_param_dtype(plan._h, dtype, master)


def _set_ls(plan):
    L = _lib()
    return L._load().gaccum_plan_set_loss_scale(plan._h, C.byref(L.LossScaleConfig()), 0x2000)


def _err():
    return _lib()._load().gaccum_last_error().decode()


def test_dtype_codes_match_the_header():
    L = _lib()
    assert (L.DTYPE_F32, L.DTYPE_BF16, L.DTYPE_F16) == (0, 1, 2)


@pytest.mark.parametrize("dtype", [1, 2])
def test_master_slab_must_be_a_16_byte_aligned_pointer(dtype):
    L = _lib()
    for bad in (0, MASTER + 4, MASTER + 8, MASTER + 2):
        assert _set(_plan(), dtype, bad) == L.EINVAL
        assert "16-byte aligned" in _err()
    assert _set(_plan(), dtype) == L.OK


@pytest.mark.parametrize("dtype", [-1, 0, 3, 16])
def test_unknown_dtypes_are_rejected(dtype):
    L = _lib()
    assert _set(_plan(), dtype) == L.EINVAL


def test_null_plan_is_rejected():
    L = _lib()
    assert L._load().gaccum_plan_set_param_dtype(None, L.DTYPE_BF16, MASTER) == L.EINVAL


@pytest.mark.parametrize("order", ["dtype_first", "loss_scale_first", "dtype_only"])
def test_refused_after_a_compute_call_and_combines_with_loss_scaling(order):
    import gaccum_b200 as g
    L = _lib()
    plan = _plan()
    if order == "loss_scale_first":
        assert _set_ls(plan) == L.OK
    assert _set(plan, L.DTYPE_F16) == L.OK
    if order == "dtype_first":
        assert _set_ls(plan) == L.OK
    assert _set(plan, L.DTYPE_BF16) == L.OK            # may be changed until the first compute call
    with pytest.raises(L.GaccumError) as e:
        plan.accumulate(g.Plan.ptr_array([0x1000, 0x2000]), 0x1000)
    assert e.value.code == L.ENODEVICE
    assert _set(plan, L.DTYPE_BF16) == L.EINVAL
    assert "before the plan's first compute call" in _err()
    assert _set_ls(plan) == L.EINVAL


def test_algorithmic_bytes_of_a_16_bit_plan():
    L = _lib()
    fp32, half = _plan(), _plan()
    P = fp32.num_elements
    assert (fp32.algorithmic_bytes(False), fp32.algorithmic_bytes(True)) == (12 * P, 36 * P)
    for dtype in (L.DTYPE_BF16, L.DTYPE_F16):
        assert _set(half, dtype) == L.OK
        assert (half.algorithmic_bytes(False), half.algorithmic_bytes(True)) == (10 * P, 36 * P)


def test_packed_data_parallel_and_host_session_refuse_a_16_bit_plan():
    import gaccum_b200 as g
    L = _lib()
    lib = L._load()
    plan = _plan()
    assert _set(plan, L.DTYPE_BF16) == L.OK
    args = g.StepArgs(*ARGS)
    with pytest.raises(L.GaccumError) as e:
        plan.step_packed(0x1000, 0x1000, 0x1000, 0x1000, 0x1000, args, 1)
    assert e.value.code == L.EINVAL and "16-bit" in str(e.value)
    comm = L.DpComm()
    comm.world, comm.rank = 2, 0
    grads = g.Plan.ptr_array([0x1000, 0x2000])
    for fn in (lib.gaccum_step_dp, lib.gaccum_apply_dp):
        assert fn(plan._h, C.byref(comm), grads, 0x1000, 0x1000, C.byref(args), 1, None) == L.EINVAL
        assert "16-bit" in _err()
    h = C.c_void_p()
    assert lib.gaccum_host_session_create(C.byref(h), plan._h) == L.EINVAL
    assert "16-bit" in _err()
    # none of the refusals counted as a compute call
    assert _set(plan, L.DTYPE_F16) == L.OK


def test_python_train_ops_refuse_16_bit_parameters():
    torch = pytest.importorskip("torch")
    import gaccum_b200 as g
    from gaccum_b200.distributed import DataParallelTrainOp, FusedDataParallelTrainOp
    from gaccum_b200.train_op import GaccumTrainOp, HostTrainOp, PackedTrainOp
    hp = g.HParams.bert()
    for dt in (torch.bfloat16, torch.float16):
        p = [torch.zeros(4, dtype=dt)]
        with pytest.raises(ValueError, match="PackedTrainOp"):
            PackedTrainOp(p, ["w"], hp, 2, lambda s: 1e-3)
        with pytest.raises(ValueError, match="HostTrainOp"):
            HostTrainOp(p, ["w"], hp, 2, lambda s: 1e-3)
        with pytest.raises(ValueError, match="multi-GPU"):
            FusedDataParallelTrainOp(p, ["w"], hp, 2, lambda s: 1e-3)

        class _Engine:               # what DataParallelTrainOp sees of a 16-bit GaccumTrainOp
            master = torch.zeros(32)
        with pytest.raises(ValueError, match="multi-GPU"):
            DataParallelTrainOp(_Engine())
    with pytest.raises(ValueError, match="mixed dtypes"):
        GaccumTrainOp([torch.zeros(4, dtype=torch.bfloat16), torch.zeros(4)], ["a", "b"], hp, 2, lambda s: 1e-3)
    with pytest.raises(ValueError, match="mixed dtypes"):
        GaccumTrainOp([torch.zeros(4, dtype=torch.bfloat16), torch.zeros(4, dtype=torch.float16)], ["a", "b"], hp, 2,
                      lambda s: 1e-3)
