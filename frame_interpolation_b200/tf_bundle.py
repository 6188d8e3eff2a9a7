"""TensorFlow-free reader (and minimal writer) for TensorBundle checkpoints -- the
`variables/variables.index` + `variables/variables.data-00000-of-00001` pair inside a TF2
SavedModel directory such as the released `pretrained_models/film_net/Style/saved_model`
(reference README.md:69-83, written by training/train_lib.py:280 /
training/build_saved_model_cli.py:73).

Format (tensorflow/core/util/tensor_bundle, tensorflow/core/lib/io/table -- a LevelDB-style
sorted string table):

  index file   = data blocks | metaindex block | index block | 48-byte footer
  block        = entries | restart offsets (u32 each) | num_restarts (u32) ; followed on disk by a
                 5-byte trailer: compression type (0 = none, 1 = snappy) + masked crc32c
  entry        = varint shared_key_len, varint unshared_key_len, varint value_len, key suffix, value
  footer       = metaindex BlockHandle, index BlockHandle (varint offset + varint size each),
                 zero padding to 40 bytes, magic 0xdb4775248b80fb57 (little-endian u64)
  index block  = entries  last_key_of_block -> BlockHandle
  data entries = ""  -> BundleHeaderProto {1: num_shards, 2: endianness, 3: version}
                 name -> BundleEntryProto {1: dtype, 2: TensorShapeProto, 3: shard_id, 4: offset,
                                           5: size, 6: crc32c (fixed32)}
  data shard   = raw little-endian tensor bytes at [offset, offset + size)

PARITY NOTE: there is no TensorFlow and no real SavedModel in the build container, so this reader
is validated only against bundles produced by `write_bundle` below (same understanding of the
format on both sides) plus hand-built byte strings in tests/test_tf_bundle.py. Snappy-compressed
blocks are not supported (TF writes bundle indices uncompressed).

Object-graph checkpoints (what `model.save` writes) key variables by attribute path, e.g.
`.../extract_sublevels/convs/3/kernel/.ATTRIBUTES/VARIABLE_VALUE`; `film_weights_from_bundle`
maps both that style (through the attribute names of the reference classes,
feature_extractor.py:117-123, pyramid_flow_estimator.py:112-123,64-83, fusion.py:62-101) and plain
variable names onto the engine's table.
"""
from __future__ import annotations

import os
import re
import struct
from typing import Dict, List, Mapping, Optional, Tuple

import numpy as np

_MAGIC = 0xDB4775248B80FB57
_DTYPES = {1: np.float32, 2: np.float64, 3: np.int32, 4: np.uint8, 9: np.int64, 19: np.float16}


# ------------------------------------------------------------------------------------------
# primitives
# ------------------------------------------------------------------------------------------
def _varint(buf: bytes, pos: int) -> Tuple[int, int]:
    out, shift = 0, 0
    while True:
        b = buf[pos]
        pos += 1
        out |= (b & 0x7F) << shift
        if not b & 0x80:
            return out, pos
        shift += 7


def _put_varint(v: int) -> bytes:
    out = bytearray()
    while True:
        b = v & 0x7F
        v >>= 7
        if v:
            out.append(b | 0x80)
        else:
            out.append(b)
            return bytes(out)


def _parse_proto(buf: bytes) -> Dict[int, list]:
    """Minimal protobuf wire parser: field number -> list of raw values (ints or bytes)."""
    out: Dict[int, list] = {}
    pos = 0
    while pos < len(buf):
        key, pos = _varint(buf, pos)
        field, wire = key >> 3, key & 7
        if wire == 0:
            v, pos = _varint(buf, pos)
        elif wire == 1:
            v = struct.unpack_from("<Q", buf, pos)[0]
            pos += 8
        elif wire == 2:
            ln, pos = _varint(buf, pos)
            v = buf[pos:pos + ln]
            pos += ln
        elif wire == 5:
            v = struct.unpack_from("<I", buf, pos)[0]
            pos += 4
        else:
            raise ValueError(f"unsupported protobuf wire type {wire}")
        out.setdefault(field, []).append(v)
    return out


def _read_block(data: bytes, offset: int, size: int) -> List[Tuple[bytes, bytes]]:
    ctype = data[offset + size]
    if ctype != 0:
        raise ValueError("compressed table block (snappy) is not supported")
    blk = data[offset:offset + size]
    (num_restarts,) = struct.unpack_from("<I", blk, size - 4)
    limit = size - 4 - 4 * num_restarts
    entries, pos, key = [], 0, b""
    while pos < limit:
        shared, pos = _varint(blk, pos)
        unshared, pos = _varint(blk, pos)
        vlen, pos = _varint(blk, pos)
        key = key[:shared] + blk[pos:pos + unshared]
        pos += unshared
        entries.append((key, blk[pos:pos + vlen]))
        pos += vlen
    return entries


# ------------------------------------------------------------------------------------------
# reader
# ------------------------------------------------------------------------------------------
def read_index(index_path: str) -> Dict[str, dict]:
    """Parses `variables.index` -> {tensor name: {dtype, shape, shard_id, offset, size}}."""
    data = open(index_path, "rb").read()
    if len(data) < 48 or struct.unpack_from("<Q", data, len(data) - 8)[0] != _MAGIC:
        raise ValueError(f"{index_path}: not a TensorBundle index (bad table magic)")
    footer = data[-48:]
    _, p = _varint(footer, 0)          # metaindex offset
    _, p = _varint(footer, p)          # metaindex size
    idx_off, p = _varint(footer, p)
    idx_size, p = _varint(footer, p)
    out: Dict[str, dict] = {}
    for _, handle in _read_block(data, idx_off, idx_size):
        off, q = _varint(handle, 0)
        size, q = _varint(handle, q)
        for key, value in _read_block(data, off, size):
            if key == b"":
                continue                                       # BundleHeaderProto
            e = _parse_proto(value)
            dims = []
            if 2 in e:
                shape = _parse_proto(e[2][0])
                for d in shape.get(2, []):
                    dims.append(_parse_proto(d).get(1, [0])[0])
            out[key.decode()] = {"dtype": e.get(1, [0])[0], "shape": tuple(int(d) for d in dims),
                                 "shard_id": e.get(3, [0])[0], "offset": e.get(4, [0])[0],
                                 "size": e.get(5, [0])[0]}
    return out


def read_bundle(prefix: str) -> Dict[str, np.ndarray]:
    """`prefix` = '<saved_model_dir>/variables/variables'. Returns every numeric tensor."""
    index = read_index(prefix + ".index")
    shards = sorted({e["shard_id"] for e in index.values()})
    nshards = max(shards) + 1 if shards else 1
    blobs: Dict[int, bytes] = {}
    out: Dict[str, np.ndarray] = {}
    for name, e in index.items():
        dt = _DTYPES.get(e["dtype"])
        if dt is None:
            continue                                           # strings (object graph proto) etc.
        sid = e["shard_id"]
        if sid not in blobs:
            path = f"{prefix}.data-{sid:05d}-of-{nshards:05d}"
            blobs[sid] = open(path, "rb").read()
        raw = blobs[sid][e["offset"]:e["offset"] + e["size"]]
        out[name] = np.frombuffer(raw, dtype=np.dtype(dt).newbyteorder("<")).reshape(e["shape"]).copy()
    return out


# ------------------------------------------------------------------------------------------
# mapping SavedModel keys -> engine weight table
# ------------------------------------------------------------------------------------------
_SUFFIX = "/.ATTRIBUTES/VARIABLE_VALUE"


def film_weights_from_bundle(tensors: Mapping[str, np.ndarray]) -> Dict[str, np.ndarray]:
    """Maps checkpoint keys to `spec.weight_table()` names. Handles (a) variable-name keys
    (`feat_net/sub_extractor/cfeat_conv_3/kernel`), (b) object-graph keys built from the
    reference's attribute names (`.../extract_sublevels/convs/3/kernel/.ATTRIBUTES/VARIABLE_VALUE`,
    `.../_predictors/1/_convs/0/bias/...`, `.../convs/2/1/kernel/...`, `.../output_conv/kernel/...`).
    Optimizer slots and non-float tensors are ignored."""
    from . import spec, weights as W
    table = dict(spec.weight_table())
    out: Dict[str, np.ndarray] = {}
    named: Dict[str, np.ndarray] = {}
    for key, arr in tensors.items():
        if arr.dtype != np.float32 or "OPTIMIZER_SLOT" in key or "optimizer" in key.lower():
            continue
        k = key[:-len(_SUFFIX)] if key.endswith(_SUFFIX) else key
        m = re.search(r"extract_sublevels/convs/(\d+)/(kernel|bias)$", k)
        if m:
            out[f"feat_net/sub_extractor/cfeat_conv_{int(m.group(1))}/{m.group(2)}"] = arr
            continue
        m = re.search(r"_predictors/(\d+)/_convs/(\d+)/(kernel|bias)$", k)
        if m:
            p = min(int(m.group(1)), spec.SPECIALIZED_LEVELS)   # levels >= 3 share one predictor object
            name = spec.FLOW_PREDICTOR_NAMES[p]
            out[f"predict_flow/{name}/conv_{int(m.group(2))}/{m.group(3)}"] = arr
            continue
        m = re.search(r"convs/(\d+)/(\d+)/(kernel|bias)$", k)      # Fusion.convs[level][j]
        if m:
            out[f"fusion/level_{int(m.group(1))}/conv_{int(m.group(2))}/{m.group(3)}"] = arr
            continue
        m = re.search(r"output_conv/(kernel|bias)$", k)
        if m:
            out[f"fusion/output_conv/{m.group(1)}"] = arr
            continue
        named[k] = arr
    if len(out) < len(table):
        # Mixed / variable-name keys: take table-named tensors directly, and resolve the fusion convs' Keras
        # auto-names (`fusion/conv2d_<n>`, a GLOBAL counter that need not start at 0) by creation order --
        # independently of each other, so one missing group cannot hide what the other one found.
        for k, v in W.from_named_arrays(named, partial=True).items():
            out.setdefault(k, v)
    missing = sorted(set(table) - set(out))
    if missing:
        raise ValueError(f"bundle does not contain the FILM variables: missing {missing[:4]} ... "
                         f"({len(missing)} of {len(table)})")
    for k, s in table.items():
        if tuple(out[k].shape) != tuple(s):
            raise ValueError(f"{k}: shape {out[k].shape} != {s}")
    return {k: np.ascontiguousarray(out[k], np.float32) for k in table}


def convert_saved_model(saved_model_dir: str, out_path: str) -> str:
    """<dir>/variables/variables.{index,data-*} -> FILMW1 file readable by film_create."""
    from . import weights as W
    prefix = os.path.join(saved_model_dir, "variables", "variables")
    W.save(out_path, film_weights_from_bundle(read_bundle(prefix)))
    return out_path


# ------------------------------------------------------------------------------------------
# minimal writer (tests, and exporting engine weights back to a TF-loadable bundle)
# ------------------------------------------------------------------------------------------
def _crc32c_table():
    t = []
    for i in range(256):
        c = i
        for _ in range(8):
            c = (c >> 1) ^ 0x82F63B78 if c & 1 else c >> 1
        t.append(c)
    return t


_CRC_T = _crc32c_table()


def crc32c(data: bytes, crc: int = 0) -> int:
    crc ^= 0xFFFFFFFF
    for b in data:
        crc = _CRC_T[(crc ^ b) & 0xFF] ^ (crc >> 8)
    return crc ^ 0xFFFFFFFF


def _mask_crc(c: int) -> int:
    return ((((c >> 15) | (c << 17)) & 0xFFFFFFFF) + 0xA282EAD8) & 0xFFFFFFFF


def _proto_field(field: int, wire: int, payload) -> bytes:
    key = _put_varint((field << 3) | wire)
    if wire == 0:
        return key + _put_varint(payload)
    if wire == 2:
        return key + _put_varint(len(payload)) + payload
    if wire == 5:
        return key + struct.pack("<I", payload)
    raise ValueError(wire)


def _build_block(entries: List[Tuple[bytes, bytes]]) -> bytes:
    body = bytearray()
    for k, v in entries:                         # restart interval 1: no key sharing
        body += _put_varint(0) + _put_varint(len(k)) + _put_varint(len(v)) + k + v
    restarts = []
    pos = 0
    for k, v in entries:
        restarts.append(pos)
        pos += len(_put_varint(0)) + len(_put_varint(len(k))) + len(_put_varint(len(v))) + len(k) + len(v)
    if not restarts:
        restarts = [0]
    for r in restarts:
        body += struct.pack("<I", r)
    body += struct.pack("<I", len(restarts))
    return bytes(body)


def write_bundle(prefix: str, tensors: Mapping[str, np.ndarray], with_crc: bool = False) -> None:
    """Writes a single-shard bundle (uncompressed index, one data block)."""
    os.makedirs(os.path.dirname(prefix) or ".", exist_ok=True)
    rev = {np.dtype(v): k for k, v in _DTYPES.items()}
    data = bytearray()
    entries: List[Tuple[bytes, bytes]] = []
    header = _proto_field(1, 0, 1) + _proto_field(3, 2, _proto_field(1, 0, 1))
    entries.append((b"", header))
    for name in sorted(tensors):
        a = np.ascontiguousarray(tensors[name])
        raw = a.astype(a.dtype.newbyteorder("<")).tobytes()
        shape = b"".join(_proto_field(2, 2, _proto_field(1, 0, int(d))) for d in a.shape)
        e = _proto_field(1, 0, rev[np.dtype(a.dtype)]) + _proto_field(2, 2, shape)
        if len(data):
            e += _proto_field(4, 0, len(data))
        e += _proto_field(5, 0, len(raw))
        if with_crc:
            e += _proto_field(6, 5, _mask_crc(crc32c(raw)))
        entries.append((name.encode(), e))
        data += raw
    with open(prefix + ".data-00000-of-00001", "wb") as f:
        f.write(bytes(data))
    out = bytearray()

    def emit(block: bytes) -> bytes:
        off = len(out)
        out.extend(block)
        out.append(0)                                           # no compression
        out.extend(struct.pack("<I", _mask_crc(crc32c(block + b"\x00"))))
        return _put_varint(off) + _put_varint(len(block))

    data_handle = emit(_build_block(entries))
    meta_handle = emit(_build_block([]))
    index_handle = emit(_build_block([(entries[-1][0], data_handle)]))
    footer = meta_handle + index_handle
    footer += b"\x00" * (40 - len(footer)) + struct.pack("<Q", _MAGIC)
    out.extend(footer)
    with open(prefix + ".index", "wb") as f:
        f.write(bytes(out))


if __name__ == "__main__":
    import sys
    if len(sys.argv) != 3:
        raise SystemExit("usage: python -m frame_interpolation_b200.tf_bundle <saved_model_dir> <out.filmw>")
    print(convert_saved_model(sys.argv[1], sys.argv[2]))
