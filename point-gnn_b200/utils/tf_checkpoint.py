"""Pure-Python reader for TensorFlow-1.x "bundle" checkpoints (no TensorFlow needed).

The reference saves its trained models with ``tf.train.Saver`` (reference
train.py:496,578-593) and run.py restores them with ``saver.restore``
(reference run.py:192-202).  On disk that is

* ``model-N.index``   - a leveldb-style sorted string table.  Key = variable
  name, value = a ``BundleEntryProto`` (dtype, shape, shard_id, offset, size,
  crc32c).  The entry with the empty key is the ``BundleHeaderProto``.
* ``model-N.data-00000-of-00001`` - the raw little-endian tensor bytes.

Only what the Point-GNN checkpoints need is implemented: uncompressed table
blocks, one shard, DT_FLOAT / DT_INT32 / DT_INT64 tensors.
"""
import os
import struct

import numpy as np

_TABLE_MAGIC = 0xDB4775248B80FB57
_DTYPES = {1: np.float32, 3: np.int32, 9: np.int64, 2: np.float64}


def _varint(buf, pos):
    result = 0
    shift = 0
    while True:
        b = buf[pos]
        pos += 1
        result |= (b & 0x7F) << shift
        if not b & 0x80:
            return result, pos
        shift += 7


def _block_handle(buf, pos):
    offset, pos = _varint(buf, pos)
    size, pos = _varint(buf, pos)
    return offset, size, pos


def _read_block(data, offset, size):
    """Return the (key, value) pairs of one table block (prefix-compressed)."""
    block = data[offset:offset + size]
    compression = data[offset + size]
    if compression != 0:
        raise ValueError('compressed checkpoint index blocks are not supported')
    num_restarts = struct.unpack('<I', block[-4:])[0]
    limit = len(block) - 4 * (num_restarts + 1)
    pos = 0
    key = b''
    out = []
    while pos < limit:
        shared, pos = _varint(block, pos)
        non_shared, pos = _varint(block, pos)
        value_len, pos = _varint(block, pos)
        key = key[:shared] + bytes(block[pos:pos + non_shared])
        pos += non_shared
        out.append((key, bytes(block[pos:pos + value_len])))
        pos += value_len
    return out


def _parse_proto(buf):
    """Minimal protobuf wire decoder -> {field_number: [values]}."""
    fields = {}
    pos = 0
    while pos < len(buf):
        tag, pos = _varint(buf, pos)
        field, wire = tag >> 3, tag & 7
        if wire == 0:
            val, pos = _varint(buf, pos)
        elif wire == 2:
            n, pos = _varint(buf, pos)
            val = bytes(buf[pos:pos + n])
            pos += n
        elif wire == 5:
            val = struct.unpack('<I', buf[pos:pos + 4])[0]
            pos += 4
        elif wire == 1:
            val = struct.unpack('<Q', buf[pos:pos + 8])[0]
            pos += 8
        else:
            raise ValueError('unsupported protobuf wire type %d' % wire)
        fields.setdefault(field, []).append(val)
    return fields


def _parse_shape(buf):
    dims = []
    for dim in _parse_proto(buf).get(2, []):      # TensorShapeProto.dim
        dims.append(_parse_proto(dim).get(1, [0])[0])   # Dim.size
    return tuple(dims)


def read_index(index_path):
    """-> {variable_name: dict(dtype, shape, shard, offset, size)}."""
    with open(index_path, 'rb') as f:
        data = f.read()
    footer = data[-48:]
    if struct.unpack('<Q', footer[-8:])[0] != _TABLE_MAGIC:
        raise ValueError('%s is not a TensorFlow checkpoint index' % index_path)
    _, _, pos = _block_handle(footer, 0)               # metaindex (unused)
    idx_off, idx_size, _ = _block_handle(footer, pos)
    entries = {}
    for _, handle in _read_block(data, idx_off, idx_size):
        off, size, _ = _block_handle(handle, 0)
        for key, value in _read_block(data, off, size):
            if key == b'':
                continue                                # BundleHeaderProto
            p = _parse_proto(value)
            entries[key.decode()] = dict(
                dtype=p.get(1, [0])[0],
                shape=_parse_shape(p[2][0]) if 2 in p else (),
                shard=p.get(3, [0])[0],
                offset=p.get(4, [0])[0],
                size=p.get(5, [0])[0],
                crc32c=p.get(6, [None])[0])         # masked CRC32C of the tensor's bytes
    return entries


def latest_checkpoint(checkpoint_dir):
    """Mirror of tf.train.latest_checkpoint: parse the ``checkpoint`` text file."""
    with open(os.path.join(checkpoint_dir, 'checkpoint')) as f:
        for line in f:
            if line.startswith('model_checkpoint_path:'):
                name = line.split(':', 1)[1].strip().strip('"')
                return os.path.join(checkpoint_dir, os.path.basename(name))
    raise FileNotFoundError('no checkpoint state in %s' % checkpoint_dir)


def load_checkpoint(prefix):
    """prefix = '<dir>/model-1400000' (or the checkpoint directory) -> {variable_name: np.ndarray}.

    A directory without TensorFlow files but with ``weights.npz`` (variable name -> array, e.g. the export that
    tools/make_golden.py writes) is accepted too."""
    if os.path.isdir(prefix):
        if not os.path.isfile(os.path.join(prefix, 'checkpoint')) and os.path.isfile(os.path.join(prefix, 'weights.npz')):
            return dict(np.load(os.path.join(prefix, 'weights.npz')))
        prefix = latest_checkpoint(prefix)
    entries = read_index(prefix + '.index')
    with open(prefix + '.data-00000-of-00001', 'rb') as f:
        blob = f.read()
    out = {}
    for name, e in entries.items():
        if e['shard'] != 0 or e['dtype'] not in _DTYPES:
            continue
        dt = np.dtype(_DTYPES[e['dtype']]).newbyteorder('<')
        arr = np.frombuffer(blob, dtype=dt, count=e['size'] // dt.itemsize,
                            offset=e['offset'])
        out[name] = arr.reshape(e['shape']).copy()
    return out
