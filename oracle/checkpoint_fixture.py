"""Rebuild the reference's trained checkpoints from the fixtures under tests/golden/ (TEST INFRASTRUCTURE).

A TF-1 bundle checkpoint is a small ``model-N.index`` table plus ``model-N.data-00000-of-00001``, the raw tensor bytes
(several MB).  tests/golden/checkpoints/<name>/ holds the reference's own ``checkpoint`` state file and ``.index`` (and,
for two checkpoints, the gzipped ``.meta`` graph); the tensors are the committed weights_<name>.npz plus the global
step ``Variable``.  rebuild() writes the data file back at the offsets the index gives and checks every tensor against
the masked CRC32C the reference's saver stored in the index, so a rebuilt checkpoint is byte for byte the shipped one.
"""
import atexit
import gzip
import json
import os
import shutil
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden')
FIXTURES = os.path.join(GOLDEN, 'checkpoints')
_DTYPES = {1: '<f4', 2: '<f8', 3: '<i4', 9: '<i8'}


def _crc32c_table():
    table = []
    for i in range(256):
        c = i
        for _ in range(8):
            c = (c >> 1) ^ 0x82F63B78 if c & 1 else c >> 1
        table.append(c)
    return table


_TABLE = _crc32c_table()


def crc32c(data):
    crc = 0xFFFFFFFF
    table = _TABLE
    for b in data:
        crc = table[(crc ^ b) & 0xFF] ^ (crc >> 8)
    return crc ^ 0xFFFFFFFF


def masked_crc32c(data):
    """TensorFlow's crc32c::Mask (tensorflow/core/lib/hash/crc32c.h)."""
    c = crc32c(data)
    return (((c >> 15) | (c << 17)) + 0xA282EAD8) & 0xFFFFFFFF


def names():
    return sorted(os.listdir(FIXTURES))


def rebuild(name, out_dir):
    """Write checkpoint directory <out_dir>/<name> (checkpoint, config, .index, .data, .meta if stored) -> its path."""
    from pointgnn_b200.utils import tf_checkpoint
    src = os.path.join(FIXTURES, name)
    dst = os.path.join(out_dir, name)
    os.makedirs(dst, exist_ok=True)
    for f in os.listdir(src):
        if f.endswith('.meta.gz'):
            with gzip.open(os.path.join(src, f), 'rb') as i, open(os.path.join(dst, f[:-3]), 'wb') as o:
                shutil.copyfileobj(i, o)
        else:
            shutil.copy(os.path.join(src, f), dst)
    with open(os.path.join(GOLDEN, 'config_%s.json' % name)) as f, open(os.path.join(dst, 'config'), 'w') as o:
        json.dump(json.load(f), o)
    prefix = tf_checkpoint.latest_checkpoint(dst)
    tensors = dict(np.load(os.path.join(GOLDEN, 'weights_%s.npz' % name)))
    tensors['Variable'] = np.int64(os.path.basename(prefix).split('-')[-1])     # the global step, model-<step>
    entries = tf_checkpoint.read_index(prefix + '.index')
    blob = bytearray(max(e['offset'] + e['size'] for e in entries.values()))
    for key, e in entries.items():
        raw = np.ascontiguousarray(tensors[key], dtype=_DTYPES[e['dtype']]).tobytes()
        if len(raw) != e['size'] or masked_crc32c(raw) != e['crc32c']:
            raise ValueError('%s: stored tensor %s does not match the checkpoint index' % (name, key))
        blob[e['offset']:e['offset'] + e['size']] = raw
    with open(prefix + '.data-00000-of-00001', 'wb') as f:
        f.write(bytes(blob))
    return dst


_cache = {}


def cached(name):
    """rebuild() into a per-process temporary directory, once per checkpoint."""
    if 'dir' not in _cache:
        _cache['dir'] = tempfile.mkdtemp(prefix='pg_ckpt_')
        atexit.register(shutil.rmtree, _cache['dir'], True)
    if name not in _cache:
        _cache[name] = rebuild(name, _cache['dir'])
    return _cache[name]
