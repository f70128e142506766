"""Weight import / export formats around the model path (SURVEY.md section 8 row f-4).

* ``read_tf_checkpoint`` -- a dependency-free reader of TensorFlow's V2 checkpoint ("tensor
  bundle"): what ``tf.train.Saver`` writes for the reference (``model.ckpt-N.index`` +
  ``model.ckpt-N.data-00000-of-00001``; restored by hdrnet/bin/run.py:136-142 and
  hdrnet/bin/freeze_graph.py:36-85).  TensorFlow is not installed here and the reference ships
  no checkpoint, so this follows the published on-disk format (tensorflow/core/util/
  tensor_bundle: an SSTable of BundleEntryProto records keyed by variable name, LevelDB table
  format, no block compression).  Pinned by a bundle assembled byte by byte from the format
  specifications by an independent script (tests/golden/make_tf_bundle_fixture.py), by the round
  trip against ``write_tf_checkpoint`` below and by every CRC-32C the format carries; it has not
  met a file produced by TensorFlow itself.
* ``model_weights`` -- variable-name filter: the reference's graph variables under
  ``inference/`` (run.py:92), optimiser slots and counters dropped.
* ``upgrade_legacy_names`` -- the old-checkpoint name map of scripts/upgrade.py:29-67.
* ``export_guide_bins`` / ``load_guide_bins`` -- the raw float32 guide parameter dumps the
  reference's freeze step writes for its GPU demo (hdrnet/bin/freeze_graph.py:105-185), incl.
  the batch-norm folding of the pointwise-NN guide.
"""
from __future__ import annotations

import os
import re
import struct

import numpy as np

# ---------------------------------------------------------------------------------------------
# CRC-32C (Castagnoli) and LevelDB's mask, as the table format stores it
# ---------------------------------------------------------------------------------------------
_CRC_TABLE = None


def _crc_table():
    global _CRC_TABLE
    if _CRC_TABLE is None:
        t = np.zeros(256, np.uint32)
        for i in range(256):
            c = i
            for _ in range(8):
                c = (c >> 1) ^ 0x82F63B78 if c & 1 else c >> 1
            t[i] = c
        _CRC_TABLE = [int(v) for v in t]
    return _CRC_TABLE


def crc32c(data: bytes, crc: int = 0) -> int:
    t = _crc_table()
    c = crc ^ 0xFFFFFFFF
    for b in data:
        c = t[(c ^ b) & 0xFF] ^ (c >> 8)
    return c ^ 0xFFFFFFFF


def _mask(crc: int) -> int:
    return (((crc >> 15) | (crc << 17)) + 0xA282EAD8) & 0xFFFFFFFF


# ---------------------------------------------------------------------------------------------
# varints / the few protobuf messages involved (hand-decoded: no generated code needed)
# ---------------------------------------------------------------------------------------------
def _get_varint(buf: bytes, pos: int):
    shift = result = 0
    while True:
        if pos >= len(buf):
            raise ValueError("truncated varint")
        b = buf[pos]
        pos += 1
        result |= (b & 0x7F) << shift
        if not b & 0x80:
            return result, pos
        shift += 7
        if shift > 63:
            raise ValueError("varint too long")


def _put_varint(v: int) -> bytes:
    out = bytearray()
    v &= (1 << 64) - 1
    while True:
        b = v & 0x7F
        v >>= 7
        if v:
            out.append(b | 0x80)
        else:
            out.append(b)
            return bytes(out)


def _pb_fields(buf: bytes):
    """Yield (field_number, wire_type, value) of one protobuf message."""
    pos = 0
    while pos < len(buf):
        key, pos = _get_varint(buf, pos)
        field, wt = key >> 3, key & 7
        if wt == 0:
            val, pos = _get_varint(buf, pos)
        elif wt == 1:
            val = buf[pos:pos + 8]
            pos += 8
        elif wt == 2:
            n, pos = _get_varint(buf, pos)
            val = buf[pos:pos + n]
            pos += n
        elif wt == 5:
            val = buf[pos:pos + 4]
            pos += 4
        else:
            raise ValueError(f"unsupported protobuf wire type {wt}")
        yield field, wt, val


# tensorflow/core/framework/types.proto
_DTYPES = {1: np.float32, 2: np.float64, 3: np.int32, 4: np.uint8, 5: np.int16, 6: np.int8,
           9: np.int64, 10: np.bool_, 17: np.uint16, 19: np.float16, 22: np.uint32, 23: np.uint64}
_DTYPE_CODES = {np.dtype(v): k for k, v in _DTYPES.items()}


def _parse_shape(buf: bytes):
    dims = []
    for field, _, val in _pb_fields(buf):
        if field == 2:                                   # repeated Dim dim = 2
            size = 0
            for f2, _, v2 in _pb_fields(val):
                if f2 == 1:                              # int64 size = 1
                    size = v2 - (1 << 64) if v2 >> 63 else v2
            dims.append(size)
        elif field == 3 and val:                         # unknown_rank
            raise ValueError("tensor of unknown rank in checkpoint")
    return tuple(dims)


def _parse_entry(buf: bytes):
    e = {"dtype": 0, "shape": (), "shard_id": 0, "offset": 0, "size": 0, "crc32c": None, "slices": 0}
    for field, wt, val in _pb_fields(buf):
        if field == 1:
            e["dtype"] = val
        elif field == 2:
            e["shape"] = _parse_shape(val)
        elif field == 3:
            e["shard_id"] = val
        elif field == 4:
            e["offset"] = val
        elif field == 5:
            e["size"] = val
        elif field == 6:
            e["crc32c"] = struct.unpack("<I", val)[0]
        elif field == 7:
            e["slices"] += 1
    return e


# ---------------------------------------------------------------------------------------------
# LevelDB table (SSTable) -- the .index file
# ---------------------------------------------------------------------------------------------
_TABLE_MAGIC = 0xDB4775248B80FB57
_FOOTER_LEN = 48


def _read_block(data: bytes, offset: int, size: int, verify: bool) -> bytes:
    if offset + size + 5 > len(data):
        raise ValueError("block handle points outside the index file")
    block = data[offset:offset + size]
    ctype = data[offset + size]
    if verify:
        stored = struct.unpack("<I", data[offset + size + 1:offset + size + 5])[0]
        if _mask(crc32c(data[offset:offset + size + 1])) != stored:
            raise ValueError("index block checksum mismatch")
    if ctype != 0:
        raise ValueError("compressed index blocks are not supported (TensorFlow writes none)")
    return block


def _block_entries(block: bytes):
    if len(block) < 4:
        raise ValueError("index block too short")
    n_restarts = struct.unpack("<I", block[-4:])[0]
    end = len(block) - 4 - 4 * n_restarts
    if end < 0:
        raise ValueError("corrupt restart array")
    pos, key = 0, b""
    while pos < end:
        shared, pos = _get_varint(block, pos)
        non_shared, pos = _get_varint(block, pos)
        vlen, pos = _get_varint(block, pos)
        key = key[:shared] + block[pos:pos + non_shared]
        pos += non_shared
        yield key, block[pos:pos + vlen]
        pos += vlen


def _read_table(path: str, verify: bool):
    with open(path, "rb") as f:
        data = f.read()
    if len(data) < _FOOTER_LEN or struct.unpack("<Q", data[-8:])[0] != _TABLE_MAGIC:
        raise ValueError(f"{path}: not a TensorFlow checkpoint index (bad table magic)")
    footer = data[-_FOOTER_LEN:]
    _, p = _get_varint(footer, 0)          # metaindex handle (unused)
    _, p = _get_varint(footer, p)
    idx_off, p = _get_varint(footer, p)
    idx_size, p = _get_varint(footer, p)
    out = []
    for _, handle in _block_entries(_read_block(data, idx_off, idx_size, verify)):
        off, q = _get_varint(handle, 0)
        size, _ = _get_varint(handle, q)
        out.extend(_block_entries(_read_block(data, off, size, verify)))
    return out


def latest_checkpoint(checkpoint_dir: str):
    """tf.train.latest_checkpoint: the prefix named by the ``checkpoint`` state file."""
    state = os.path.join(checkpoint_dir, "checkpoint")
    if not os.path.exists(state):
        return None
    with open(state) as f:
        for line in f:
            m = re.match(r'\s*model_checkpoint_path:\s*"(.*)"\s*$', line)
            if m:
                p = m.group(1)
                return p if os.path.isabs(p) else os.path.join(checkpoint_dir, p)
    return None


def read_tf_checkpoint(prefix: str, verify: bool = True) -> dict:
    """{variable name: ndarray} of a V2 checkpoint given its prefix (``.../model.ckpt-N``) or
    the directory holding a ``checkpoint`` state file.  ``verify`` checks the block and tensor
    CRC-32Cs (pure Python: about a second per MB of tensor data)."""
    if os.path.isdir(prefix):
        p = latest_checkpoint(prefix)
        if p is None:
            raise FileNotFoundError(f"no checkpoint state file in {prefix}")
        prefix = p
    entries = _read_table(prefix + ".index", verify)
    if not entries or entries[0][0] != b"":
        raise ValueError("checkpoint index has no header entry")
    num_shards, little_endian = 1, True
    for field, _, val in _pb_fields(entries[0][1]):      # BundleHeaderProto
        if field == 1:
            num_shards = val
        elif field == 2:
            little_endian = (val == 0)
    if not little_endian:
        raise ValueError("big-endian checkpoints are not supported")
    shards = {}
    out = {}
    for key, val in entries[1:]:
        e = _parse_entry(val)
        name = key.decode("utf-8")
        if e["slices"]:
            raise ValueError(f"{name}: partitioned variables are not supported")
        if e["dtype"] not in _DTYPES:
            raise ValueError(f"{name}: unsupported dtype code {e['dtype']}")
        sid = e["shard_id"]
        if sid not in shards:
            path = f"{prefix}.data-{sid:05d}-of-{num_shards:05d}"
            with open(path, "rb") as f:
                shards[sid] = f.read()
        raw = shards[sid][e["offset"]:e["offset"] + e["size"]]
        dt = np.dtype(_DTYPES[e["dtype"]])
        n = int(np.prod(e["shape"], dtype=np.int64)) if e["shape"] else 1
        if len(raw) != e["size"] or n * dt.itemsize != e["size"]:
            raise ValueError(f"{name}: data size {e['size']} does not match shape {e['shape']}")
        if verify and e["crc32c"] is not None and _mask(crc32c(raw)) != e["crc32c"]:
            raise ValueError(f"{name}: tensor checksum mismatch")
        out[name] = np.frombuffer(raw, dtype=dt).reshape(e["shape"]).copy()
    return out


# ---------------------------------------------------------------------------------------------
# Writer of the same format (export; and what the reader is tested against)
# ---------------------------------------------------------------------------------------------
def _shape_proto(shape) -> bytes:
    out = bytearray()
    for d in shape:
        dim = b"\x08" + _put_varint(int(d))
        out += b"\x12" + _put_varint(len(dim)) + dim
    return bytes(out)


def _entry_proto(dtype_code, shape, offset, size, crc) -> bytes:
    out = bytearray()
    out += b"\x08" + _put_varint(dtype_code)
    sp = _shape_proto(shape)
    out += b"\x12" + _put_varint(len(sp)) + sp
    if offset:
        out += b"\x20" + _put_varint(offset)             # shard_id 0 and offset 0 are defaults
    out += b"\x28" + _put_varint(size)
    out += b"\x35" + struct.pack("<I", crc)
    return bytes(out)


class _BlockBuilder:
    def __init__(self, restart_interval=16):
        self.buf, self.restarts, self.count, self.last = bytearray(), [0], 0, b""
        self.interval = restart_interval

    def add(self, key: bytes, value: bytes):
        shared = 0
        if self.count % self.interval == 0 and self.count:
            self.restarts.append(len(self.buf))
        elif self.count:
            m = min(len(key), len(self.last))
            while shared < m and key[shared] == self.last[shared]:
                shared += 1
        self.buf += _put_varint(shared) + _put_varint(len(key) - shared) + _put_varint(len(value))
        self.buf += key[shared:] + value
        self.last, self.count = key, self.count + 1

    def finish(self) -> bytes:
        return bytes(self.buf) + b"".join(struct.pack("<I", r) for r in self.restarts) + \
            struct.pack("<I", len(self.restarts))


def write_tf_checkpoint(prefix: str, tensors: dict, block_size: int = 4096) -> None:
    """Write {name: ndarray} as a single-shard V2 checkpoint plus the ``checkpoint`` state file."""
    os.makedirs(os.path.dirname(os.path.abspath(prefix)), exist_ok=True)
    items = []
    offset = 0
    with open(prefix + ".data-00000-of-00001", "wb") as f:
        for name in sorted(tensors, key=lambda s: s.encode("utf-8")):
            a = np.asarray(tensors[name])
            if not a.flags.c_contiguous:                           # (ascontiguousarray makes 0-d 1-d)
                a = np.ascontiguousarray(a)
            if a.dtype not in _DTYPE_CODES:
                raise ValueError(f"{name}: dtype {a.dtype} has no checkpoint encoding here")
            raw = a.astype(a.dtype.newbyteorder("<"), copy=False).tobytes()
            f.write(raw)
            items.append((name.encode("utf-8"),
                          _entry_proto(_DTYPE_CODES[a.dtype], a.shape, offset, len(raw), _mask(crc32c(raw)))))
            offset += len(raw)
    header = b"\x08\x01" + b"\x1a\x02\x08\x01"            # num_shards = 1, version { producer = 1 }
    records = [(b"", header)] + items

    out = bytearray()
    index = _BlockBuilder(restart_interval=1)

    def flush(block: _BlockBuilder):
        body = block.finish()
        handle = _put_varint(len(out)) + _put_varint(len(body))
        out.extend(body + b"\x00" + struct.pack("<I", _mask(crc32c(body + b"\x00"))))
        return handle

    cur = _BlockBuilder()
    for key, val in records:
        cur.add(key, val)
        if len(cur.buf) >= block_size:
            index.add(cur.last, flush(cur))
            cur = _BlockBuilder()
    if cur.count:
        index.add(cur.last, flush(cur))
    meta_handle = flush(_BlockBuilder())                 # empty metaindex block
    index_handle = flush(index)
    footer = meta_handle + index_handle
    footer += b"\x00" * (40 - len(footer)) + struct.pack("<Q", _TABLE_MAGIC)
    out.extend(footer)
    with open(prefix + ".index", "wb") as f:
        f.write(bytes(out))
    with open(os.path.join(os.path.dirname(os.path.abspath(prefix)), "checkpoint"), "w") as f:
        base = os.path.basename(prefix)
        f.write(f'model_checkpoint_path: "{base}"\nall_model_checkpoint_paths: "{base}"\n')


# ---------------------------------------------------------------------------------------------
# Variable names
# ---------------------------------------------------------------------------------------------
_SLOT = re.compile(r"/(Adam(_\d+)?|Momentum|RMSProp(_\d+)?|ExponentialMovingAverage)$")


def model_weights(variables: dict) -> dict:
    """The graph variables the inference models read (scope ``inference/``, run.py:92), as
    float32; optimiser slots, ``global_step`` and the Adam power accumulators are dropped."""
    out = {}
    for name, val in variables.items():
        name = name[:-2] if name.endswith(":0") else name
        if not name.startswith("inference/") or _SLOT.search(name):
            continue
        out[name] = np.asarray(val, np.float32)
    return out


# scripts/upgrade.py:29-67: checkpoints written before the graph was re-scoped.
_LEGACY_SPLAT = {"conv1": ("biases",), "conv2": ("BatchNorm/beta",), "conv3": ("BatchNorm/beta",),
                 "conv4": ("BatchNorm/beta",)}


def legacy_name_map() -> dict:
    m = {}
    for conv, (bias,) in _LEGACY_SPLAT.items():
        m[f"{conv}/weights"] = f"inference/coefficients/splat/{conv}/weights"
        m[f"{conv}/biases"] = f"inference/coefficients/splat/{conv}/{bias}"
    for layer in ("conv1", "conv2", "fc1", "fc2"):
        m[f"global_{layer}/weights"] = f"inference/coefficients/global/{layer}/weights"
        m[f"global_{layer}/biases"] = f"inference/coefficients/global/{layer}/BatchNorm/beta"
    m["global_fc3/weights"] = "inference/coefficients/global/fc3/weights"
    m["grid_conv1/weights"] = "inference/coefficients/local/conv1/weights"
    m["grid_conv1/biases"] = "inference/coefficients/local/conv1/BatchNorm/beta"
    m["grid_conv2/weights"] = "inference/coefficients/local/conv2/weights"
    m["post_fusion_conv/weights"] = "inference/coefficients/prediction/conv1/weights"
    m["post_fusion_conv/biases"] = "inference/coefficients/prediction/conv1/biases"
    m["guide/guide/ccm"] = "inference/guide/ccm"
    m["guide/guide/ccm_bias"] = "inference/guide/ccm_bias"
    for leaf in ("shifts", "slopes", "channel_mixing/weights", "channel_mixing/biases"):
        m[f"guide/{leaf}"] = f"inference/guide/{leaf}"
    return m


def upgrade_legacy_names(variables: dict) -> dict:
    """Old variable names -> the ``inference/...`` names (scripts/upgrade.py:29-61); the two old
    biases that fed the fusion sum are ADDED into the single fc3 bias (upgrade.py:63-67).

    The new graph is a batch-norm graph: the old biases become ``BatchNorm/beta``.  The reference
    builds that graph and runs its initialiser before assigning the transferred tensors, so every
    batch-normed layer also has ``moving_mean`` = 0 and ``moving_variance`` = 1 (the
    tf.contrib.layers.batch_norm initial values) -- emitted here, or the upgraded weights would not
    load (models._fold needs them; load the result with params['batch_norm'] = True)."""
    m = legacy_name_map()
    out = {}
    for name, val in variables.items():
        name = name[:-2] if name.endswith(":0") else name
        if name in m:
            out[m[name]] = np.asarray(val, np.float32)
            if m[name].endswith("/BatchNorm/beta"):
                scope = m[name][:-len("/beta")]
                out[scope + "/moving_mean"] = np.zeros_like(out[m[name]])
                out[scope + "/moving_variance"] = np.ones_like(out[m[name]])
    fused = [np.asarray(variables[k], np.float32) for k in ("grid_conv2/biases", "global_fc3/biases")
             if k in variables]
    if fused:
        out["inference/coefficients/global/fc3/biases"] = sum(fused[1:], fused[0])
    return out


# ---------------------------------------------------------------------------------------------
# Raw float32 guide dumps (freeze_graph.py:105-185)
# ---------------------------------------------------------------------------------------------
_BN_EPS = 1e-3   # tf.contrib.layers.batch_norm default epsilon (the 'batchnorm/add/y' constant)


def _fold_nn_guide(w, prefix):
    c1w = np.asarray(w[f"{prefix}/conv1/weights"], np.float32)
    beta = np.asarray(w[f"{prefix}/conv1/BatchNorm/beta"], np.float32)
    mu = np.asarray(w[f"{prefix}/conv1/BatchNorm/moving_mean"], np.float32)
    var = np.asarray(w[f"{prefix}/conv1/BatchNorm/moving_variance"], np.float32)
    s = np.sqrt(var + np.float32(_BN_EPS))
    c1b = (beta - mu / s).astype(np.float32)                       # freeze_graph.py:166
    c1w = np.squeeze((c1w / s).astype(np.float32))                 # [3, F]
    conv1 = np.vstack([c1w, c1b[np.newaxis, :]])                   # [4, F]
    conv2 = np.append(np.squeeze(np.asarray(w[f"{prefix}/conv2/weights"], np.float32)),
                      np.squeeze(np.asarray(w[f"{prefix}/conv2/biases"], np.float32)))
    return conv1.T.astype(np.float32), conv2.astype(np.float32)    # files hold conv1.T, conv2


def guide_bins(weights: dict, model_name: str) -> dict:
    """{file name: float32 array} exactly as freeze_graph.py lays them out."""
    g = "inference/guide"
    if model_name == "HDRNetCurves":
        ccm34 = np.vstack((weights[f"{g}/ccm"], np.asarray(weights[f"{g}/ccm_bias"])[np.newaxis, :]))
        mixw = np.squeeze(np.asarray(weights[f"{g}/channel_mixing/weights"], np.float32))
        mixb = np.asarray(weights[f"{g}/channel_mixing/biases"], np.float32).reshape(-1)
        return {
            "guide_ccm_f32_3x4.bin": np.asarray(ccm34, np.float32).T,
            "guide_shifts_f32_16x3.bin": np.squeeze(np.asarray(weights[f"{g}/shifts"], np.float32)).T,
            "guide_slopes_f32_16x3.bin": np.squeeze(np.asarray(weights[f"{g}/slopes"], np.float32)).T,
            "guide_mix_matrix_f32_1x4.bin": np.append(mixw, mixb[0]).astype(np.float32),
        }
    if model_name == "HDRNetPointwiseNNGuide":
        c1, c2 = _fold_nn_guide(weights, g)
        return {"guide_conv1.bin": c1, "guide_conv2.bin": c2}
    if model_name == "HDRNetGaussianPyrNN":
        out = {}
        for lvl in range(3):
            c1, c2 = _fold_nn_guide(weights, f"{g}/level_{lvl}")
            out[f"guide_level{lvl}_conv1.bin"] = c1
            out[f"guide_level{lvl}_conv2.bin"] = c2
        return out
    if model_name == "HDRNetGaussianPyr":
        raise ValueError("HDRNetGaussianPyr has no guide dumps: freeze_graph.py has no layout for its three curves "
                         "guides (checkpoint.freeze_model writes its frozen model file)")
    raise ValueError(f"unknown model {model_name}")


def export_guide_bins(weights: dict, model_name: str, out_dir: str) -> list:
    os.makedirs(out_dir, exist_ok=True)
    paths = []
    for fname, arr in guide_bins(weights, model_name).items():
        path = os.path.join(out_dir, fname)
        with open(path, "wb") as f:
            f.write(np.ascontiguousarray(arr, np.float32).tobytes())
        paths.append(path)
    return paths


def load_guide_bins(bin_dir: str, model_name: str, feats: int = 16) -> dict:
    """Read the dumps back into ready-to-use guide parameters (batch norm already folded):
    curves: ccm [3,3] (in, out), ccm_bias [3], shifts / slopes [3,16], mix [3], mix_bias;
    NN guides: w1 [3,F], b1 [F], w2 [F], b2 (per level for the pyramid model)."""
    def rd(name):
        return np.fromfile(os.path.join(bin_dir, name), dtype="<f4")

    if model_name == "HDRNetCurves":
        ccm43 = rd("guide_ccm_f32_3x4.bin").reshape(3, 4).T        # file = [out][in + bias]
        mix = rd("guide_mix_matrix_f32_1x4.bin")
        return {"ccm": ccm43[:3].copy(), "ccm_bias": ccm43[3].copy(),
                "shifts": rd("guide_shifts_f32_16x3.bin").reshape(16, 3).T.copy(),
                "slopes": rd("guide_slopes_f32_16x3.bin").reshape(16, 3).T.copy(),
                "mix": mix[:3].copy(), "mix_bias": float(mix[3])}

    def nn(c1name, c2name):
        c1 = rd(c1name).reshape(feats, 4)                          # conv1.T: [F][3 weights + bias]
        c2 = rd(c2name)
        return {"w1": c1[:, :3].T.copy(), "b1": c1[:, 3].copy(), "w2": c2[:feats].copy(),
                "b2": float(c2[feats])}

    if model_name == "HDRNetPointwiseNNGuide":
        return nn("guide_conv1.bin", "guide_conv2.bin")
    if model_name == "HDRNetGaussianPyrNN":
        return {f"level_{l}": nn(f"guide_level{l}_conv1.bin", f"guide_level{l}_conv2.bin") for l in range(3)}
    raise ValueError(f"unknown model {model_name}")


# ---------------------------------------------------------------------------------------------
# model_params out of the meta graph (hdrnet/bin/train.py:60-63, hdrnet/utils.py:19-23)
# ---------------------------------------------------------------------------------------------
# train.py stores every model parameter as a Const node and lists the nodes in the graph
# collection 'model_params'; run.py / freeze_graph.py import the .meta file and evaluate them.
# The messages involved (public .proto definitions): MetaGraphDef{graph_def=2, collection_def=4},
# GraphDef{node=1}, NodeDef{name=1, op=2, attr=5}, AttrValue{tensor=8}, TensorProto{dtype=1,
# tensor_content=4, float_val=5, double_val=6, int_val=7, string_val=8, int64_val=10,
# bool_val=11}, CollectionDef{node_list=1}, NodeList{value=1}.  Pinned like the bundle reader: by a
# MetaGraphDef assembled from the .proto definitions by an independent script
# (tests/golden/make_tf_meta_fixture.py: packed scalars, tensor_content, negative varints, other
# nodes / collections to skip); it has not met a file produced by TensorFlow itself.
def _map_entry(buf: bytes):
    key = val = b""
    for field, _, v in _pb_fields(buf):
        if field == 1:
            key = v
        elif field == 2:
            val = v
    return key.decode("utf-8"), val


def _scalars(val, wt, kind):
    if wt == 2:                                            # packed repeated
        if kind == "varint":
            out, pos = [], 0
            while pos < len(val):
                v, pos = _get_varint(val, pos)
                out.append(v)
            return out
        fmt = {"f32": "<f", "f64": "<d"}[kind]
        n = struct.calcsize(fmt)
        return [struct.unpack(fmt, val[i:i + n])[0] for i in range(0, len(val), n)]
    if kind == "varint":
        return [val]
    return [struct.unpack({"f32": "<f", "f64": "<d"}[kind], val)[0]]


def _const_value(tensor: bytes):
    dtype, content, vals, strings, shape = 0, None, [], [], ()
    for field, wt, v in _pb_fields(tensor):
        if field == 1:
            dtype = v
        elif field == 2:
            shape = _parse_shape(v)
        elif field == 4:
            content = v
        elif field == 5:
            vals += _scalars(v, wt, "f32")
        elif field == 6:
            vals += _scalars(v, wt, "f64")
        elif field in (7, 10):
            vals += [x - (1 << 64) if x >> 63 else x for x in _scalars(v, wt, "varint")]
        elif field == 11:
            vals += [bool(x) for x in _scalars(v, wt, "varint")]
        elif field == 8:
            strings.append(v.decode("utf-8"))
    n = int(np.prod(shape, dtype=np.int64)) if shape else 1
    if strings:
        out = strings
    elif content is not None and dtype in _DTYPES:
        out = np.frombuffer(content, dtype=np.dtype(_DTYPES[dtype])).reshape(-1).tolist()
    else:
        out = vals or [False if dtype == 10 else 0]       # proto3 default: zero / False
        if dtype == 10:
            out = [bool(x) for x in out]
        elif dtype in (1, 2, 19):
            out = [float(x) for x in out]
    out = list(out) + [out[-1]] * max(0, n - len(out))    # a repeated tail value is stored once
    return out[:n] if shape else out[0]


def read_meta_model_params(meta_path: str) -> dict:
    """{parameter name: python value} of the 'model_params' collection of a ``.meta`` file."""
    with open(meta_path, "rb") as f:
        meta = f.read()
    graph, wanted = b"", []
    for field, _, val in _pb_fields(meta):
        if field == 2:
            graph = val
        elif field == 4:
            key, cdef = _map_entry(val)
            if key == "model_params":
                for f1, _, node_list in _pb_fields(cdef):
                    if f1 == 1:
                        wanted += [v.decode("utf-8").split(":")[0] for f2, _, v in _pb_fields(node_list) if f2 == 1]
    if not wanted:
        raise ValueError(f"{meta_path}: no 'model_params' collection")
    out = {}
    for field, _, node in _pb_fields(graph):
        if field != 1:
            continue
        name, attrs = "", {}
        for f1, _, v in _pb_fields(node):
            if f1 == 1:
                name = v.decode("utf-8")
            elif f1 == 5:
                k, a = _map_entry(v)
                attrs[k] = a
        if name in wanted and "value" in attrs:
            for f2, _, v in _pb_fields(attrs["value"]):
                if f2 == 8:
                    out[name] = _const_value(v)
    missing = [n for n in wanted if n not in out]
    if missing:
        raise ValueError(f"{meta_path}: model_params nodes without a constant value: {missing}")
    return out


def import_checkpoint(checkpoint_dir: str, verify: bool = False, legacy: bool = False):
    """(params, weights) of a TensorFlow training directory: latest checkpoint -> inference
    variables; ``<prefix>.meta`` -> model_params when the file is there (else params is None)."""
    prefix = latest_checkpoint(checkpoint_dir) if os.path.isdir(checkpoint_dir) else checkpoint_dir
    if prefix is None:
        raise FileNotFoundError(f"could not find a checkpoint in {checkpoint_dir}")
    variables = read_tf_checkpoint(prefix, verify=verify)
    weights = upgrade_legacy_names(variables) if legacy else model_weights(variables)
    params = read_meta_model_params(prefix + ".meta") if os.path.exists(prefix + ".meta") else None
    return params, weights


# ---------------------------------------------------------------------------------------------
# Frozen model file: the arrays the kernels consume, for the whole-model C-ABI (hdrnet_model_create)
# ---------------------------------------------------------------------------------------------
# Layout (little-endian; csrc/model.cu and DESIGN.md row f-12 describe the same bytes):
#   char[8] magic | u32 version | u32 kind | i32 net_input_size, spatial_bin, luma_bins,
#   channel_multiplier, guide width | u32 array count | per array: u32 ndim, u32 dims[ndim],
#   float32 data | u32 CRC-32C of every byte before it.
FROZEN_MAGIC = b"HDRNETFZ"
FROZEN_VERSION = 1
FROZEN_KINDS = ("HDRNetCurves", "HDRNetPointwiseNNGuide", "HDRNetGaussianPyrNN")   # kind = index
# Every model a frozen file holds, kind = index (HDRNET_MODEL_*): FROZEN_KINDS, the first three kinds,
# then HDRNetGaussianPyr (3).  FROZEN_KINDS keeps naming the first three for callers that describe only those.
FROZEN_MODEL_NAMES = FROZEN_KINDS + ("HDRNetGaussianPyr",)
_CURVES_GUIDE_MODELS = ("HDRNetCurves", "HDRNetGaussianPyr")   # guide width 16: the curves' knots
_FROZEN_HEADER = struct.Struct("<8sII5iI")


def frozen_arrays(weights: dict, params: dict) -> list:
    """The arrays of the frozen file, in its order, as float32 numpy: each coefficient-network layer's
    weights and bias (an empty array for a layer without one) as ``models._Prepared`` builds them --
    batch norm folded by ``models._fold`` -- then the guide: the curves guide's ccm, ccm_bias, shifts,
    slopes, mix and [mix_bias] of each curves guide, or the folded w1, b1, w2 and [b2] of each
    pointwise-NN guide (one guide per pyramid level)."""
    import torch

    from . import models
    name = params.get("model_name", "HDRNetCurves")
    if name not in FROZEN_MODEL_NAMES:
        raise ValueError(f"model_name {name!r} is not one of {FROZEN_MODEL_NAMES}")
    prep = models._Prepared(weights, params, torch.device("cpu"), getattr(models, name)._nn_guide)
    out = []
    for scope, _, _ in models._coefficient_specs(params):
        w, b, _ = prep.layers[scope]
        out.append(w.detach().numpy())
        out.append(np.zeros(0, np.float32) if b is None else b.detach().numpy())
    for g in prep.guides:
        if isinstance(g, models._CurvesGuide):
            out += [g.ccm, g.ccm_bias, g.shifts, g.slopes, g.mix, np.array([g.mix_bias], np.float32)]
        else:
            out += [g.w1, g.b1, g.w2, np.array([g.b2], np.float32)]
    return [np.ascontiguousarray(a, np.float32) for a in out]


def _frozen_bytes(kind: int, hyper, arrays) -> bytes:
    parts = [_FROZEN_HEADER.pack(FROZEN_MAGIC, FROZEN_VERSION, kind, *hyper, len(arrays))]
    for a in arrays:
        parts.append(struct.pack(f"<I{a.ndim}I", a.ndim, *a.shape))
        parts.append(np.ascontiguousarray(a, "<f4").tobytes())
    body = b"".join(parts)
    return body + struct.pack("<I", crc32c(body))


def freeze_model(weights: dict, params: dict, path: str) -> str:
    """Write the frozen model file of (weights, params) to `path`: what hdrnet_model_create (and
    ``hdrnet_b200.frozen.FrozenModel``, and the ``hdrnet_run`` program) load.  Returns `path`."""
    arrays = frozen_arrays(weights, params)
    name = params.get("model_name", "HDRNetCurves")
    width = 16 if name in _CURVES_GUIDE_MODELS else int(arrays[-4].shape[1])
    hyper = (int(params["net_input_size"]), int(params["spatial_bin"]), int(params["luma_bins"]),
             int(params["channel_multiplier"]), width)
    data = _frozen_bytes(FROZEN_MODEL_NAMES.index(name), hyper, arrays)
    with open(path, "wb") as f:
        f.write(data)
    return path


def read_frozen_model(path: str) -> dict:
    """A frozen model file back: ``model_name``, ``net_input_size``, ``spatial_bin``, ``luma_bins``,
    ``channel_multiplier``, ``guide_width`` and ``arrays`` (the list frozen_arrays gave).  Raises
    ValueError for a wrong magic, version, length or CRC-32C (shapes are the C side's to check)."""
    with open(path, "rb") as f:
        data = f.read()
    if len(data) < _FROZEN_HEADER.size + 4 or data[:8] != FROZEN_MAGIC:
        raise ValueError(f"{path}: not a frozen hdrnet_b200 model")
    magic, version, kind, S, sb, gd, cm, width, n = _FROZEN_HEADER.unpack_from(data)
    if version != FROZEN_VERSION:
        raise ValueError(f"{path}: frozen model format version {version}, this reader knows {FROZEN_VERSION}")
    if crc32c(data[:-4]) != struct.unpack_from("<I", data, len(data) - 4)[0]:
        raise ValueError(f"{path}: CRC-32C mismatch")
    if kind >= len(FROZEN_MODEL_NAMES):
        raise ValueError(f"{path}: unknown model kind {kind}")
    arrays, off = [], _FROZEN_HEADER.size
    end = len(data) - 4
    for _ in range(n):
        if off + 4 > end:
            raise ValueError(f"{path}: truncated array header")
        (ndim,) = struct.unpack_from("<I", data, off)
        if off + 4 + 4 * ndim > end:
            raise ValueError(f"{path}: truncated array header")
        shape = struct.unpack_from(f"<{ndim}I", data, off + 4)
        off += 4 + 4 * ndim
        count = int(np.prod(shape, dtype=np.int64))
        if off + 4 * count > end:
            raise ValueError(f"{path}: truncated array")
        arrays.append(np.frombuffer(data, "<f4", count, off).reshape(shape).astype(np.float32))
        off += 4 * count
    if off != end:
        raise ValueError(f"{path}: {end - off} bytes after the last array")
    return dict(model_name=FROZEN_MODEL_NAMES[kind], net_input_size=S, spatial_bin=sb, luma_bins=gd,
                channel_multiplier=cm, guide_width=width, arrays=arrays)
