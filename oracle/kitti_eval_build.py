"""Compile the reference's KITTI evaluator into oracle/_ref/evaluate_object_3d_offline.

The binary is the reference evaluator with a convex-polygon stand-in for Boost.Geometry (oracle/boost_standin/):
kitti_native_evaluation/src/evaluate_object_3d_offline.cpp is compiled unmodified from the reference tree against
those headers.  Rectangle intersections agree with Boost up to rounding; they are not bit-identical.

Without a reference tree this does nothing: an existing binary is kept and nothing fails.
"""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
REFERENCE_ROOT = '/root/reference'
STANDIN = os.path.join(HERE, 'boost_standin')
BINARY = os.path.join(HERE, '_ref', 'evaluate_object_3d_offline')


def build(reference_root=REFERENCE_ROOT):
    """-> path of the binary, or None when there is neither a reference tree nor an earlier build."""
    src = os.path.join(reference_root, 'kitti_native_evaluation', 'src', 'evaluate_object_3d_offline.cpp')
    if not os.path.isfile(src):
        return BINARY if os.path.isfile(BINARY) else None
    inputs = [src] + [os.path.join(d, f) for d, _, fs in os.walk(STANDIN) for f in fs]
    if os.path.isfile(BINARY) and os.path.getmtime(BINARY) >= max(os.path.getmtime(p) for p in inputs):
        return BINARY
    os.makedirs(os.path.dirname(BINARY), exist_ok=True)
    subprocess.run(['g++', '-O2', '-std=c++17', '-w', '-I', STANDIN,
                    '-I', os.path.join(reference_root, 'kitti_native_evaluation', 'include'), src, '-o', BINARY],
                   check=True)
    return BINARY


def binary():
    """The compiled evaluator, or None."""
    return BINARY if os.path.isfile(BINARY) else None
