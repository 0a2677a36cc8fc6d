"""The apply kernels in the built libgaccum.so are exactly the ones the dispatch matrix launches (no GPU needed).

``tests/test_gpu_apply_matrix.py`` runs one case per dispatch key and ``tests/apply_matrix.py`` maps each case to the
kernel instantiation ``gaccum_abi.cu`` launches for it.  Here the ``__global__`` entries of the library (``cuobjdump
-symbols`` | ``cu++filt``) are compared with that mapping: a new template flag, an instantiation the dispatch cannot
reach, or a dispatch key the matrix does not run fails without a GPU.  The schedule constants the edge tests aim at are
read out of csrc/*.cuh the same way.
"""
import os
import re
import shutil
import subprocess

import pytest

from apply_matrix import LAYOUTS, Schedule, instantiation, matrix_cases

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "gradient-accumulation-tf-estimator_b200", "csrc")
APPLY_KERNELS = ("apply_kernel", "apply_clip_kernel", "lamb_apply_kernel")
# every other __global__ entry point of the library, with its number of instantiations
OTHER_KERNELS = {"accumulate_kernel": 10, "dp_apply_kernel": 4, "ema_init_kernel": 1, "loss_scale_init_kernel": 1}


def _constants():
    """``constexpr int kName = <expr>;`` of csrc/*.cuh, evaluated in order (integer arithmetic)."""
    env = {}
    for f in sorted(os.listdir(CSRC)):
        if not f.endswith(".cuh"):
            continue
        with open(os.path.join(CSRC, f)) as fh:
            for m in re.finditer(r"^constexpr int (k\w+) = ([^;]+);", fh.read(), re.M):
                expr = m.group(2).replace("/", "//")
                if re.fullmatch(r"[\w\s()*+\-/]+", expr):
                    env[m.group(1)] = eval(expr, {"__builtins__": {}}, dict(env))
    return env


def _tool(name):
    from gaccum_b200 import build
    for cand in (os.path.join(os.path.dirname(build.nvcc_path()), name), shutil.which(name)):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError(f"{name} not found next to nvcc")


def _entries():
    """(template name, template arguments) of every __global__ function in the library."""
    from gaccum_b200 import _lib
    sym = subprocess.run([_tool("cuobjdump"), "-symbols", _lib.lib_path()], check=True, capture_output=True, text=True).stdout
    mangled = [ln.split()[-1] for ln in sym.splitlines() if "STT_FUNC" in ln and "STO_ENTRY" in ln]
    assert mangled, "no __global__ functions found in the library"
    names = subprocess.run([_tool("cu++filt")], input="\n".join(mangled) + "\n", check=True, capture_output=True,
                           text=True).stdout.split("\n")[:len(mangled)]
    out = []
    for n in names:
        m = re.match(r"(?:void )?gaccum::(\w+)(?:<([^>]*)>)?\(", n)   # a template's name carries its return type
        assert m, n
        args = tuple(int(v) for v in re.findall(r"\((?:int|bool)\)(-?\d+)", m.group(2) or ""))
        out.append((m.group(1), args))
    return out


def test_schedule_constants_match_the_kernels():
    c = _constants()
    assert c["kTile"] == Schedule.TILE
    assert c["kGroups"] == Schedule.GROUPS
    assert c["kStashTiles"] == Schedule.STASH_TILES[False]
    assert c["kLambBlocksPerSm"] == Schedule.LAMB_BLOCKS_PER_SM
    # ClipLayout<true>: a pass-2 slot of 5 streams; the stash gets what the ring leaves of the same shared memory
    p2 = 5 * (c["kTile"] // 4)
    ring_bytes = c["kGroups"] * max(c["kP1Slots"] * c["kP1SlotVecs"], p2) * 16
    assert (c["kClipSmemBytes"] - ring_bytes) // (c["kGroups"] * c["kTile"] * 4) == Schedule.STASH_TILES[True]


def test_matrix_covers_every_apply_instantiation_with_or_without_gradients():
    consts = _constants()
    cases = matrix_cases()
    assert len(cases) == 336 and len(set(cases)) == 336
    claimed = {instantiation(c, consts) for c in cases}
    entries = _entries()
    built = [e for e in entries if e[0] in APPLY_KERNELS]
    assert len(built) == len(set(built)), "an apply instantiation appears twice"
    assert set(built) == claimed, (sorted(set(built) - claimed), sorted(claimed - set(built)))
    # bf16 and fp16 share their instantiations: 5 (CAP, H) pairs x 2 (EMA) x (2 + 6 + 4) kernels
    assert len(claimed) == 5 * 2 * 12 == 120
    # a case without gradients runs the kernel of the same case with them
    for c in cases:
        assert instantiation(c, consts) == instantiation(c._replace(has_g=not c.has_g), consts)
    others = {}
    for name, _ in entries:
        if name not in APPLY_KERNELS:
            others[name] = others.get(name, 0) + 1
    assert others == OTHER_KERNELS


@pytest.mark.parametrize("layout", sorted(LAYOUTS))
def test_every_layout_reaches_its_own_24_instantiations(layout):
    """Different layouts of one (CAP, H) pair -- bf16 and fp16 -- map to the same kernels, all others to disjoint ones."""
    consts = _constants()
    mine = {instantiation(c, consts) for c in matrix_cases() if c.layout == layout}
    assert len(mine) == 24
    for other in LAYOUTS:
        theirs = {instantiation(c, consts) for c in matrix_cases() if c.layout == other}
        if LAYOUTS[other][:2] == LAYOUTS[layout][:2]:
            assert theirs == mine
        else:
            assert not theirs & mine
