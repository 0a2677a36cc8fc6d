"""TensorFlow checkpoint (V2 "tensor bundle") files under the reference's variable names -- SURVEY.md 8(f) #3.

The reference keeps its whole optimizer state in TF variables, so ``tf.estimator`` / ``tf.train.Saver`` checkpoints it:
the parameters, ``global_step``, one UNNAMED ``tf.Variable`` per trainable variable for the accumulators
(optimization.py:78, 02:54, another-example.py:133 -- TensorFlow names them ``Variable``, ``Variable_1``, ... in creation =
``tf.trainable_variables()`` order), and the optimizer's slots: ``<name>/adam_m``, ``<name>/adam_v`` for
``AdamWeightDecayOptimizer`` (optimization.py:137-148), ``<name>/Adam``, ``<name>/Adam_1``, ``beta1_power``,
``beta2_power`` for ``tf.train.AdamOptimizer`` (02:41, another-example.py:135), ``<name>/lamb_m``, ``<name>/lamb_v`` and
the beta powers for LAMB.  A run that was checkpointed by the reference
mid-window can therefore be continued by this train_op, and the other way round, if those files can be read and written.

File format (restated from TensorFlow's published sources, tensorflow/core/util/tensor_bundle/ and core/lib/io/table*):
  ``<prefix>.data-00000-of-00001``  the tensors' little-endian bytes back to back, in key order
  ``<prefix>.index``                a LevelDB-format immutable table (prefix-compressed blocks with restart points every 16
                                    keys, 5-byte block trailers = compression type + masked CRC-32C, metaindex block, index
                                    block, 48-byte footer ending in the magic 0xdb4775248b80fb57), uncompressed, mapping
                                    ""  -> BundleHeaderProto {num_shards: 1, version {producer: 1}}
                                    key -> BundleEntryProto {dtype, shape, shard_id, offset, size, crc32c}
  ``checkpoint``                    text CheckpointState naming the latest prefix

NOT VERIFIED AGAINST TENSORFLOW: there is no TensorFlow (and no TF-written checkpoint) in this image.  What the tests
pin: CRC-32C against the RFC 3720 vectors, the container's invariants (magic, trailers, restart arrays, header bytes),
write -> read round trips at one and many blocks, name mapping both ways for both optimizer variants, and a GPU run that
is interrupted mid-window, saved in this format, restored into a fresh train_op and continues bit-identically.

Host-side file I/O only; nothing here touches the device path.
"""
from __future__ import annotations

import os
import struct
from typing import Dict, Iterable, List, Optional, Sequence, Tuple

import numpy as np

# ---------------------------------------------------------------------------------------------------------------------
# CRC-32C (Castagnoli), vectorised: K chunks advance together, then are folded with the "append L zero bytes" operator
# ---------------------------------------------------------------------------------------------------------------------
_POLY = 0x82F63B78


def _make_table() -> np.ndarray:
    t = np.arange(256, dtype=np.uint32)
    for _ in range(8):
        t = np.where(t & 1, (t >> 1) ^ np.uint32(_POLY), t >> 1).astype(np.uint32)
    return t


_TABLE = _make_table()
_TABLE_LIST = [int(x) for x in _TABLE]


def _raw_serial(state: int, data: bytes) -> int:
    for b in data:
        state = _TABLE_LIST[(state ^ b) & 0xFF] ^ (state >> 8)
    return state


def _zero_operator(nbytes: int) -> np.ndarray:
    """Images of the 32 basis registers after nbytes zero bytes (the register update is linear over GF(2))."""
    basis = (np.uint32(1) << np.arange(32, dtype=np.uint32)).astype(np.uint32)
    for _ in range(nbytes):
        basis = _TABLE[basis & np.uint32(0xFF)] ^ (basis >> np.uint32(8))
    return basis


def _apply(op: np.ndarray, state: int) -> int:
    out = 0
    i = 0
    while state:
        if state & 1:
            out ^= int(op[i])
        state >>= 1
        i += 1
    return out


def crc32c(data) -> int:
    """CRC-32C of a bytes-like object or a C-contiguous numpy array (iSCSI polynomial, init/xorout 0xFFFFFFFF)."""
    buf = np.frombuffer(memoryview(data).cast("B"), dtype=np.uint8) if not isinstance(data, np.ndarray) \
        else np.ascontiguousarray(data).view(np.uint8).reshape(-1)
    n = buf.size
    state = 0xFFFFFFFF
    if n >= 1 << 16:
        lanes = 1 << 14
        length = n // lanes
        cols = np.ascontiguousarray(buf[:lanes * length].reshape(lanes, length).T)    # byte j of every chunk, contiguous
        regs = np.zeros(lanes, dtype=np.uint32)                      # init 0 per chunk: the fold below supplies the real init
        for j in range(length):
            regs = _TABLE[(regs ^ cols[j]) & np.uint32(0xFF)] ^ (regs >> np.uint32(8))
        op = _zero_operator(length)
        for r in regs:
            state = _apply(op, state) ^ int(r)
        buf = buf[lanes * length:]
    state = _raw_serial(state, buf.tobytes())
    return state ^ 0xFFFFFFFF


def masked_crc32c(data) -> int:
    """TensorFlow / LevelDB store CRCs rotated and offset (crc32c::Mask), so a CRC of data that embeds CRCs stays useful."""
    c = crc32c(data)
    return (((c >> 15) | (c << 17)) + 0xA282EAD8) & 0xFFFFFFFF


# ---------------------------------------------------------------------------------------------------------------------
# protobuf wire format, the three messages needed
# ---------------------------------------------------------------------------------------------------------------------
def _varint(v: int) -> bytes:
    if v < 0:
        v += 1 << 64
    out = bytearray()
    while True:
        b = v & 0x7F
        v >>= 7
        out.append(b | (0x80 if v else 0))
        if not v:
            return bytes(out)


def _read_varint(buf: bytes, pos: int) -> Tuple[int, int]:
    shift = v = 0
    while True:
        b = buf[pos]
        pos += 1
        v |= (b & 0x7F) << shift
        if not b & 0x80:
            return v, pos
        shift += 7


_DTYPES = {1: np.dtype("<f4"), 2: np.dtype("<f8"), 3: np.dtype("<i4"), 9: np.dtype("<i8"), 10: np.dtype("bool")}   # types.proto
_DTYPE_ENUM = {v: k for k, v in _DTYPES.items()}
_HEADER = b"\x08\x01" + b"\x1a\x02\x08\x01"          # BundleHeaderProto: num_shards = 1, (endianness LITTLE = 0 omitted), version {producer: 1}


def _entry_proto(arr: np.ndarray, offset: int, crc: int) -> bytes:
    shape = b"".join(b"\x12" + _varint(len(d)) + d for d in (b"\x08" + _varint(int(s)) for s in arr.shape))   # TensorShapeProto.dim{size}
    out = b"\x08" + _varint(_DTYPE_ENUM[arr.dtype])
    out += b"\x12" + _varint(len(shape)) + shape
    if offset:
        out += b"\x20" + _varint(offset)
    if arr.nbytes:
        out += b"\x28" + _varint(arr.nbytes)
    out += b"\x35" + struct.pack("<I", crc)
    return out


def _parse_fields(buf: bytes) -> List[Tuple[int, int, object]]:
    pos, out = 0, []
    while pos < len(buf):
        key, pos = _read_varint(buf, pos)
        field, wire = key >> 3, key & 7
        if wire == 0:
            v, pos = _read_varint(buf, pos)
        elif wire == 2:
            n, pos = _read_varint(buf, pos)
            v = buf[pos:pos + n]
            pos += n
        elif wire == 5:
            v = struct.unpack_from("<I", buf, pos)[0]
            pos += 4
        elif wire == 1:
            v = struct.unpack_from("<Q", buf, pos)[0]
            pos += 8
        else:
            raise ValueError(f"unsupported protobuf wire type {wire}")
        out.append((field, wire, v))
    return out


def _parse_entry(buf: bytes) -> dict:
    e = {"dtype": 0, "shape": [], "shard_id": 0, "offset": 0, "size": 0, "crc32c": None, "slices": 0}
    for field, _, v in _parse_fields(buf):
        if field == 1:
            e["dtype"] = v
        elif field == 2:
            for f2, _, dim in _parse_fields(v):
                if f2 == 2:
                    size = 0
                    for f3, _, x in _parse_fields(dim):
                        if f3 == 1:
                            size = x
                    e["shape"].append(size)
        elif field == 3:
            e["shard_id"] = v
        elif field == 4:
            e["offset"] = v
        elif field == 5:
            e["size"] = v
        elif field == 6:
            e["crc32c"] = v
        elif field == 7:
            e["slices"] += 1
    return e


# ---------------------------------------------------------------------------------------------------------------------
# the LevelDB-format table that is the .index file
# ---------------------------------------------------------------------------------------------------------------------
_MAGIC = 0xDB4775248B80FB57
_BLOCK_SIZE = 262144           # tensorflow/core/lib/io/table_options.h
_RESTART_INTERVAL = 16


class _BlockBuilder:
    def __init__(self, restart_interval: int):
        self.interval = restart_interval
        self.buf = bytearray()
        self.restarts = [0]
        self.count = 0
        self.last = b""

    def add(self, key: bytes, value: bytes) -> None:
        shared = 0
        if self.count < self.interval:
            m = min(len(key), len(self.last))
            while shared < m and key[shared] == self.last[shared]:
                shared += 1
        else:
            self.restarts.append(len(self.buf))
            self.count = 0
        self.buf += _varint(shared) + _varint(len(key) - shared) + _varint(len(value)) + key[shared:] + value
        self.last = key
        self.count += 1

    def size(self) -> int:
        return len(self.buf) + 4 * len(self.restarts) + 4

    def empty(self) -> bool:
        return not self.buf

    def finish(self) -> bytes:
        return bytes(self.buf) + b"".join(struct.pack("<I", r) for r in self.restarts) + struct.pack("<I", len(self.restarts))


def _write_table(path: str, items: Sequence[Tuple[bytes, bytes]]) -> None:
    """items sorted by key (bytewise), keys unique."""
    out = bytearray()

    def emit(block: bytes) -> bytes:
        handle = _varint(len(out)) + _varint(len(block))
        out.extend(block)
        out.extend(b"\x00" + struct.pack("<I", masked_crc32c(block + b"\x00")))       # type 0 = kNoCompression
        return handle

    index = _BlockBuilder(1)
    data = _BlockBuilder(_RESTART_INTERVAL)
    for key, value in items:
        data.add(key, value)
        if data.size() >= _BLOCK_SIZE:
            index.add(data.last, emit(data.finish()))          # any separator in [last key, next key) is valid; the last key is one
            data = _BlockBuilder(_RESTART_INTERVAL)
    if not data.empty():
        index.add(data.last, emit(data.finish()))
    meta_handle = emit(_BlockBuilder(_RESTART_INTERVAL).finish())
    index_handle = emit(index.finish())
    footer = meta_handle + index_handle
    out.extend(footer + b"\x00" * (40 - len(footer)) + struct.pack("<Q", _MAGIC))
    with open(path, "wb") as f:
        f.write(out)


def _read_block(buf: bytes, offset: int, size: int, verify: bool) -> List[Tuple[bytes, bytes]]:
    block, trailer = buf[offset:offset + size], buf[offset + size:offset + size + 5]
    if len(trailer) != 5:
        raise ValueError("truncated table block")
    if trailer[0] != 0:
        raise ValueError(f"table block compression type {trailer[0]} not supported (TensorFlow writes bundles uncompressed)")
    if verify and struct.unpack("<I", trailer[1:])[0] != masked_crc32c(block + trailer[:1]):
        raise ValueError("table block checksum mismatch")
    n_restarts = struct.unpack_from("<I", block, len(block) - 4)[0]
    end = len(block) - 4 - 4 * n_restarts
    pos, key, out = 0, b"", []
    while pos < end:
        shared, pos = _read_varint(block, pos)
        non_shared, pos = _read_varint(block, pos)
        vlen, pos = _read_varint(block, pos)
        key = key[:shared] + block[pos:pos + non_shared]
        pos += non_shared
        out.append((key, block[pos:pos + vlen]))
        pos += vlen
    return out


def _read_table(path: str, verify: bool = True) -> List[Tuple[bytes, bytes]]:
    with open(path, "rb") as f:
        buf = f.read()
    if len(buf) < 48 or struct.unpack("<Q", buf[-8:])[0] != _MAGIC:
        raise ValueError(f"{path}: not a TensorFlow V2 checkpoint index (bad table magic)")
    footer = buf[-48:-8]
    _, pos = _read_varint(footer, 0)
    _, pos = _read_varint(footer, pos)                 # metaindex handle: unused
    ioff, pos = _read_varint(footer, pos)
    isize, pos = _read_varint(footer, pos)
    out = []
    for _, handle in _read_block(buf, ioff, isize, verify):
        off, p = _read_varint(handle, 0)
        size, _ = _read_varint(handle, p)
        out.extend(_read_block(buf, off, size, verify))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# bundles
# ---------------------------------------------------------------------------------------------------------------------
def write_bundle(prefix: str, tensors: Dict[str, np.ndarray]) -> None:
    """Write ``prefix.index`` + ``prefix.data-00000-of-00001`` holding `tensors` (name -> array), as BundleWriter does."""
    os.makedirs(os.path.dirname(os.path.abspath(prefix)), exist_ok=True)
    items: List[Tuple[bytes, bytes]] = [(b"", _HEADER)]
    offset = 0
    tmp = prefix + ".data-00000-of-00001.tmp"
    with open(tmp, "wb") as f:
        for name in sorted(tensors, key=lambda s: s.encode()):
            if not name:
                raise ValueError("the empty key is the bundle header")
            arr = np.asarray(tensors[name], order="C")            # (ascontiguousarray would turn a scalar into shape [1])
            if arr.dtype.byteorder == ">":
                arr = arr.astype(arr.dtype.newbyteorder("<"))
            if arr.dtype not in _DTYPE_ENUM:
                raise TypeError(f"{name}: dtype {arr.dtype} not supported")
            f.write(arr.tobytes())
            items.append((name.encode(), _entry_proto(arr, offset, masked_crc32c(arr))))
            offset += arr.nbytes
    os.replace(tmp, prefix + ".data-00000-of-00001")
    _write_table(prefix + ".index.tmp", items)
    os.replace(prefix + ".index.tmp", prefix + ".index")


def read_bundle(prefix: str, verify: bool = True) -> Dict[str, np.ndarray]:
    """Read every tensor of a V2 checkpoint (all shards) into numpy arrays; `verify` checks block and tensor CRCs."""
    items = _read_table(prefix + ".index", verify)
    if not items or items[0][0] != b"":
        raise ValueError(f"{prefix}.index has no bundle header")
    header = {f: v for f, _, v in _parse_fields(items[0][1])}
    num_shards = header.get(1, 0)
    if header.get(2, 0) != 0:
        raise ValueError("big-endian bundles are not supported")
    shards: Dict[int, np.memmap] = {}
    out: Dict[str, np.ndarray] = {}
    for key, value in items[1:]:
        e = _parse_entry(value)
        name = key.decode()
        if e["slices"]:
            raise ValueError(f"{name}: partitioned (sliced) variables are not supported")
        if e["dtype"] not in _DTYPES:
            raise TypeError(f"{name}: DataType {e['dtype']} not supported")
        sid = e["shard_id"]
        if sid not in shards:
            shards[sid] = np.memmap(f"{prefix}.data-{sid:05d}-of-{num_shards:05d}", dtype=np.uint8, mode="r")
        raw = np.asarray(shards[sid][e["offset"]:e["offset"] + e["size"]])
        dt = _DTYPES[e["dtype"]]
        if raw.size != e["size"] or e["size"] != int(np.prod(e["shape"], dtype=np.int64)) * dt.itemsize:
            raise ValueError(f"{name}: entry size {e['size']} does not match shape {e['shape']}")
        if verify and e["crc32c"] is not None and masked_crc32c(raw) != e["crc32c"]:
            raise ValueError(f"{name}: tensor checksum mismatch")
        out[name] = raw.view(dt).reshape(e["shape"]).copy()
    return out


def write_checkpoint_state(model_dir: str, prefix_basename: str, all_paths: Optional[Iterable[str]] = None) -> None:
    """The text ``checkpoint`` file tf.train.latest_checkpoint() reads (CheckpointState)."""
    paths = list(all_paths) if all_paths is not None else [prefix_basename]
    with open(os.path.join(model_dir, "checkpoint"), "w") as f:
        f.write(f'model_checkpoint_path: "{prefix_basename}"\n')
        for p in paths:
            f.write(f'all_model_checkpoint_paths: "{p}"\n')


def latest_checkpoint(model_dir: str) -> Optional[str]:
    try:
        with open(os.path.join(model_dir, "checkpoint")) as f:
            for line in f:
                if line.startswith("model_checkpoint_path:"):
                    p = line.split(":", 1)[1].strip().strip('"')
                    return p if os.path.isabs(p) else os.path.join(model_dir, p)
    except FileNotFoundError:
        return None
    return None


# ---------------------------------------------------------------------------------------------------------------------
# the reference's variable names  <->  this train_op's state_dict()
# ---------------------------------------------------------------------------------------------------------------------
ADAM_WEIGHT_DECAY, ADAM, LAMB = 0, 1, 2
# optimization.py:137-148 / TF1 AdamOptimizer slots / LAMB's slots, named like AdamWeightDecay's (NVIDIA's TF BERT)
_SLOTS = {ADAM_WEIGHT_DECAY: ("/adam_m", "/adam_v"), ADAM: ("/Adam", "/Adam_1"), LAMB: ("/lamb_m", "/lamb_v")}
_BETA_POWERS = (ADAM, LAMB)      # variants that keep TF1's beta1_power / beta2_power


_EMA, _EMA_STEP = "/ExponentialMovingAverage", "ExponentialMovingAverage/num_updates"
# the running total weight of the current window (a train op with window_weight=True): an fp32 scalar
_WINDOW_WEIGHT = "gradient_accumulation/window_weight"


def _accum_name(i: int) -> str:
    return "Variable" if i == 0 else f"Variable_{i}"             # unnamed tf.Variable, uniquified by the graph (optimization.py:78)


def to_reference_names(state: Dict[str, object], names: Sequence[str], variant: int) -> Dict[str, np.ndarray]:
    """train_op.state_dict() -> {reference Saver key: numpy array}.  `names` in tf.trainable_variables() order."""
    def arr(x, dt=None):
        a = x.detach().cpu().numpy() if hasattr(x, "detach") else np.asarray(x)
        return a.astype(dt) if dt is not None else a
    m_s, v_s = _SLOTS[variant]
    out = {"global_step": arr(state["global_step"], np.int64)}
    for i, n in enumerate(names):
        out[n] = arr(state[n])
        out[n + m_s] = arr(state[n + "/adam_m"])
        out[n + v_s] = arr(state[n + "/adam_v"])
        out[_accum_name(i)] = arr(state[n + "/accum_grad"])
    if variant in _BETA_POWERS:
        out["beta1_power"] = arr(state["beta1_power"], np.float32)
        out["beta2_power"] = arr(state["beta2_power"], np.float32)
    if _EMA_STEP in state:                                        # tf.train.ExponentialMovingAverage's shadow variables
        for n in names:
            out[n + _EMA] = arr(state[n + _EMA])
        out[_EMA_STEP] = arr(state[_EMA_STEP], np.int64)
    if _WINDOW_WEIGHT in state:
        out[_WINDOW_WEIGHT] = arr(state[_WINDOW_WEIGHT], np.float32).reshape(())
    return out


def from_reference_names(tensors: Dict[str, np.ndarray], names: Sequence[str], variant: int, strict: bool = True,
                         ema: bool = False, window_weight: bool = False) -> Dict[str, np.ndarray]:
    """{reference Saver key: array} -> the dictionary train_op.load_state_dict() takes.  A checkpoint written before the
    optimizer existed (a pre-trained BERT: parameters only) loads with strict=False: moments and accumulators stay zero.
    The moving averages (``<var>/ExponentialMovingAverage``, ``ExponentialMovingAverage/num_updates``) are taken when
    present, and required in strict mode when ``ema`` is True (a train op that keeps them).  The window's running weight
    (``gradient_accumulation/window_weight``, fp32) likewise, required in strict mode when ``window_weight`` is True."""
    m_s, v_s = _SLOTS[variant]
    out: Dict[str, np.ndarray] = {"global_step": np.asarray(tensors.get("global_step", 0), dtype=np.int64)}
    for i, n in enumerate(names):
        for src, dst in ((n, n), (n + m_s, n + "/adam_m"), (n + v_s, n + "/adam_v"), (_accum_name(i), n + "/accum_grad")):
            if src in tensors:
                out[dst] = tensors[src]
            elif strict:
                raise KeyError(f"checkpoint has no tensor {src!r}")
    if variant in _BETA_POWERS:
        for k in ("beta1_power", "beta2_power"):
            if k in tensors:
                out[k] = tensors[k]
            elif strict:
                raise KeyError(f"checkpoint has no tensor {k!r}")
    for k in [n + _EMA for n in names] + [_EMA_STEP]:
        if k in tensors:
            out[k] = tensors[k]
        elif strict and ema:
            raise KeyError(f"checkpoint has no tensor {k!r}")
    if _WINDOW_WEIGHT in tensors:
        out[_WINDOW_WEIGHT] = np.asarray(tensors[_WINDOW_WEIGHT], np.float32).reshape(())
    elif strict and window_weight:
        raise KeyError(f"checkpoint has no tensor {_WINDOW_WEIGHT!r}")
    return out


# ---------------------------------------------------------------------------------------------------------------------
# the reference's per-variable state  <->  the TensorFlow shim's three packed variables (tf_shim/optimization.py)
# ---------------------------------------------------------------------------------------------------------------------
def _slab_offsets(sizes: Sequence[int]) -> Tuple[List[int], int]:
    """Slab layout of include/gaccum.h (gaccum_offsets): every tensor starts at a multiple of 32 elements."""
    offs, o = [], 0
    for n in sizes:
        offs.append(o)
        o += (int(n) + 31) // 32 * 32
    return offs, o


def to_shim_names(ref: Dict[str, np.ndarray], names: Sequence[str], variant: int, betas=(0.9, 0.999)) -> Dict[str, np.ndarray]:
    """{reference Saver key: array} -> what a Saver over the shim's graph holds: the parameters and ``global_step``
    unchanged, ``gaccum/accum_grads`` / ``gaccum/adam_m`` / ``gaccum/adam_v`` packed, ``gaccum/beta_powers``.
    Lets a checkpoint written by a reference run (mid-window included) be restored into the shim's graph."""
    m_s, v_s = _SLOTS[variant]
    sizes = [int(np.asarray(ref[n]).size) for n in names]
    offs, total = _slab_offsets(sizes)
    out = {n: np.asarray(ref[n]) for n in names}
    out["global_step"] = np.asarray(ref.get("global_step", 0), dtype=np.int64)
    for slab, key in (("gaccum/accum_grads", None), ("gaccum/adam_m", m_s), ("gaccum/adam_v", v_s)):
        buf = np.zeros(total, np.float32)
        for i, n in enumerate(names):
            src = _accum_name(i) if key is None else n + key
            if src in ref:                                         # a slot the optimizer has not created yet stays zero
                buf[offs[i]:offs[i] + sizes[i]] = np.asarray(ref[src], np.float32).reshape(-1)
        out[slab] = buf
    out["gaccum/beta_powers"] = np.asarray([ref.get("beta1_power", betas[0]), ref.get("beta2_power", betas[1])], np.float32) \
        if variant in _BETA_POWERS else np.asarray(betas, np.float32)
    return out


def from_shim_names(shim: Dict[str, np.ndarray], names: Sequence[str], variant: int) -> Dict[str, np.ndarray]:
    """Inverse of to_shim_names(): a checkpoint of the shim's graph -> the reference's Saver keys."""
    m_s, v_s = _SLOTS[variant]
    sizes = [int(np.asarray(shim[n]).size) for n in names]
    offs, total = _slab_offsets(sizes)
    out = {n: np.asarray(shim[n]) for n in names}
    out["global_step"] = np.asarray(shim["global_step"], dtype=np.int64)
    for slab, key in (("gaccum/accum_grads", None), ("gaccum/adam_m", m_s), ("gaccum/adam_v", v_s)):
        buf = np.asarray(shim[slab], np.float32).reshape(-1)
        if buf.size != total:
            raise ValueError(f"{slab} holds {buf.size} elements, the variables need {total}")
        for i, n in enumerate(names):
            out[_accum_name(i) if key is None else n + key] = buf[offs[i]:offs[i] + sizes[i]].reshape(np.asarray(shim[n]).shape).copy()
    if variant in _BETA_POWERS:
        bp = np.asarray(shim["gaccum/beta_powers"], np.float32).reshape(-1)
        out["beta1_power"], out["beta2_power"] = np.float32(bp[0]), np.float32(bp[1])
    return out


def _engine_of(train_op):
    """The object that knows the variable names and the optimizer variant (wrappers keep it in .engine)."""
    eng = train_op
    while not hasattr(eng, "names") and hasattr(eng, "engine"):
        eng = eng.engine
    return eng


def save(model_dir: str, train_op, names: Optional[Sequence[str]] = None, basename: str = "model.ckpt") -> str:
    """Write ``model_dir/model.ckpt-<global_step>.{index,data-00000-of-00001}`` + ``checkpoint`` from a train_op
    (anything with state_dict(), and .names / .hp.variant on it or on its .engine).  Under data parallelism
    state_dict() is collective (moments gathered, accumulators summed: 04:55) -- every rank calls save(), rank 0
    writes, and all ranks leave together."""
    eng = _engine_of(train_op)
    names = list(names if names is not None else eng.names)
    state = train_op.state_dict()
    step = int(state["global_step"])
    prefix = os.path.join(model_dir, f"{basename}-{step}")
    comm = train_op if hasattr(train_op, "world") else getattr(train_op, "dp", None)     # optimization.TrainOp keeps its DP wrapper in .dp
    group = getattr(comm, "group", None)
    world = getattr(comm, "world", 1) if comm is not None else 1
    rank = 0
    if world > 1:
        import torch.distributed as dist
        rank = dist.get_rank(group)
    if rank == 0:
        write_bundle(prefix, to_reference_names(state, names, int(eng.hp.variant)))
        write_checkpoint_state(model_dir, os.path.basename(prefix))
    if world > 1:
        dist.barrier(group=group)
    return prefix


def restore(prefix_or_dir: str, train_op, names: Optional[Sequence[str]] = None, strict: bool = True) -> str:
    """Load a V2 checkpoint (a prefix, or a model_dir whose ``checkpoint`` file names one) into a train_op."""
    import torch
    prefix = latest_checkpoint(prefix_or_dir) if os.path.isdir(prefix_or_dir) else prefix_or_dir
    if prefix is None:
        raise FileNotFoundError(f"no checkpoint state in {prefix_or_dir}")
    eng = _engine_of(train_op)
    names = list(names if names is not None else eng.names)
    sd = from_reference_names(read_bundle(prefix), names, int(eng.hp.variant), strict, getattr(eng, "ema", None) is not None,
                              getattr(eng, "window_weight", None) is not None)
    train_op.load_state_dict({k: torch.from_numpy(np.array(v, order="C")) for k, v in sd.items()}, strict)
    return prefix


def _main(argv: Optional[Sequence[str]] = None) -> int:
    """python -m gaccum_b200.tf_checkpoint list <prefix|model_dir>
       python -m gaccum_b200.tf_checkpoint convert {to-shim|to-reference} <in prefix> <out prefix> --names FILE [--variant 0|1|2]
    (FILE: one trainable-variable name per line, in tf.trainable_variables() order -- the order is not in a checkpoint)"""
    import argparse
    ap = argparse.ArgumentParser(prog="gaccum_b200.tf_checkpoint", description=_main.__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    sub = ap.add_subparsers(dest="cmd", required=True)
    ls = sub.add_parser("list")
    ls.add_argument("prefix")
    cv = sub.add_parser("convert")
    cv.add_argument("direction", choices=["to-shim", "to-reference"])
    cv.add_argument("src")
    cv.add_argument("dst")
    cv.add_argument("--names", required=True)
    cv.add_argument("--variant", type=int, default=0, choices=[0, 1, 2])
    a = ap.parse_args(argv)
    if a.cmd == "list":
        prefix = latest_checkpoint(a.prefix) if os.path.isdir(a.prefix) else a.prefix
        if prefix is None:
            print(f"no checkpoint state in {a.prefix}")
            return 1
        for k, v in sorted(read_bundle(prefix).items(), key=lambda kv: kv[0].encode()):
            print(f"{k} ({v.dtype.name}) {list(v.shape)}")
        return 0
    with open(a.names) as f:
        names = [ln.strip() for ln in f if ln.strip()]
    src = read_bundle(a.src)
    write_bundle(a.dst, to_shim_names(src, names, a.variant) if a.direction == "to-shim" else from_shim_names(src, names, a.variant))
    return 0


if __name__ == "__main__":
    raise SystemExit(_main())
