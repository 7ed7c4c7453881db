"""ctypes binding of libpointgnn_b200.so, read from its C header include/pointgnn_b200.h.

The header is the only place the ABI is written down.  At import this module parses it - every ``PG_API`` prototype
and every integer ``#define PG_*``, which become the module's ``PG_*`` constants - without loading the library, so
CPU-only imports work.  The library is loaded on first use and the load fails loudly when it is missing or lacks a
symbol: there is no CPU or PyTorch fallback behind these wrappers.

Every wrapper calls the library through ``_call``, by the header's parameter names.  Arguments are converted by their
declared type: a device pointer takes a contiguous CUDA tensor of the pointee's dtype, a ``_host`` pointer a
contiguous NumPy array, a ctypes array or a ``byref``; only pointers, sizes and the current CUDA stream cross the
boundary.
"""
import ctypes
import os
import re

import numpy as np
import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libpointgnn_b200.so')
HEADER_PATH = os.path.join(os.path.dirname(_HERE), 'include', 'pointgnn_b200.h')

c_i64 = ctypes.c_int64
c_i32 = ctypes.c_int32


def parse_header(text):
    """-> (prototypes, constants) of C header text: {name: (return type, ((parameter type, parameter name), ...))}
    for every PG_API declaration, types spelt as ``const float* const*``, and {name: value} for every integer
    ``#define PG_*``.  Raises ImportError for a PG_API declaration it cannot read."""
    text = re.sub(r'/\*.*?\*/|//[^\n]*', ' ', text, flags=re.S)
    constants = {}
    for name, value in re.findall(r'^[ \t]*#[ \t]*define[ \t]+(PG_\w+)[ \t]+'
                                  r'(-?\w+|\([ \t]*-?\w+[ \t]*\))[ \t]*$', text, re.M):
        try:
            constants[name] = int(value.strip('() \t'), 0)
        except ValueError:     # PG_API and other non-integer macros
            pass
    text = re.sub(r'^[ \t]*#[^\n]*', ' ', text, flags=re.M)

    def spell(c_type):
        return re.sub(r'\s*\*', '*', ' '.join(c_type.split()))

    prototypes = {}
    for decl in re.findall(r'\bPG_API\b([^;]*);', text):
        m = re.fullmatch(r'\s*(.+?)\s*\b(pg_\w+)\s*\((.*)\)\s*', decl, re.S)
        params = [] if m is None or m.group(3).strip() == 'void' else [
            re.fullmatch(r'(.*?\S)\s*\b(\w+)', ' '.join(p.split())) for p in m.group(3).split(',')]
        if m is None or None in params:
            raise ImportError('%s: cannot read the declaration "PG_API %s"' % (HEADER_PATH, ' '.join(decl.split())))
        prototypes[m.group(2)] = (spell(m.group(1)), tuple((spell(p.group(1)), p.group(2)) for p in params))
    return prototypes, constants


# ---------------------------------------------------------------------------------------------
# argument conversion by declared type: convert(value, parameter name) -> what ctypes passes
# ---------------------------------------------------------------------------------------------
_RETURN_TYPES = {'int': ctypes.c_int, 'int64_t': ctypes.c_int64, 'const char*': ctypes.c_char_p}
_SCALAR_TYPES = {'int32_t': ctypes.c_int32, 'int64_t': ctypes.c_int64, 'uint32_t': ctypes.c_uint32,
                 'double': ctypes.c_double}
_DEVICE_DTYPES = {'float': torch.float32, 'double': torch.float64, 'int32_t': torch.int32, 'uint8_t': torch.uint8}
_HOST_TYPES = {'float': ctypes.c_float, 'double': ctypes.c_double, 'int32_t': ctypes.c_int32, 'int64_t': ctypes.c_int64}
_BYREF = type(ctypes.byref(ctypes.c_int()))


def _device(dtype):
    def convert(t, name):
        if t is None:
            return None
        if not isinstance(t, torch.Tensor) or not t.is_cuda:
            raise TypeError('%s must be a CUDA tensor (there is no CPU path)' % name)
        if t.dtype != dtype:
            raise TypeError('%s must be %s, got %s' % (name, dtype, t.dtype))
        if not t.is_contiguous():
            raise ValueError('%s must be contiguous' % name)
        return t.data_ptr()
    return convert


_device_f32 = _device(torch.float32)


def _host(ctype):
    pointer, dtype = ctypes.POINTER(ctype), np.dtype(ctype)

    def convert(a, name):
        if a is None:
            return None
        if isinstance(a, np.ndarray):
            if a.dtype != dtype or not a.flags.c_contiguous:
                raise TypeError('%s must be a contiguous %s array, got %s' % (name, dtype, a.dtype))
            return a.ctypes.data_as(pointer)
        if (isinstance(a, ctypes.Array) and a._type_ is ctype) or (type(a) is _BYREF and type(a._obj) is ctype):
            return a
        raise TypeError('%s must be a host %s array (NumPy, ctypes or byref), got %s' % (name, dtype, type(a).__name__))
    return convert


def _device_pointer_array(t, name):
    """const float* const*: a sequence of CUDA float32 tensors -> a host array of their device pointers."""
    return (ctypes.c_void_p * len(t))(*[_device_f32(x, name) for x in t])


def _layer(handle, name):
    if not isinstance(handle, ctypes.c_void_p):
        raise TypeError('%s must be a PreparedLayer handle' % name)
    return handle


def _layer_out(ref, name):
    if type(ref) is not _BYREF or type(ref._obj) is not ctypes.c_void_p:
        raise TypeError('%s must be byref(ctypes.c_void_p())' % name)
    return ref


def _stream(stream, name):
    """The current torch stream unless a torch.cuda.Stream is given."""
    return (torch.cuda.current_stream() if stream is None else stream).cuda_stream


_FIXED_TYPES = {      # c type -> (argtype, converter); None converter: ctypes converts the Python value
    'const float* const*': (ctypes.POINTER(ctypes.c_void_p), _device_pointer_array),
    'const pg_layer*': (ctypes.c_void_p, _layer),
    'pg_layer*': (ctypes.c_void_p, _layer),
    'pg_layer**': (ctypes.POINTER(ctypes.c_void_p), _layer_out),
}
_FIXED_TYPES.update({t: (ctype, None) for t, ctype in _SCALAR_TYPES.items()})


def _parameter(function, c_type, name):
    """-> (argtype, converter) of one parameter; ImportError for a type the binding does not know."""
    if c_type in _FIXED_TYPES:
        return _FIXED_TYPES[c_type]
    if c_type == 'void*' and name == 'stream':
        return ctypes.c_void_p, _stream
    m = re.fullmatch(r'(?:const )?(\w+)\*', c_type)
    if m and name.endswith('_host') and m.group(1) in _HOST_TYPES:
        ctype = _HOST_TYPES[m.group(1)]
        return ctypes.POINTER(ctype), _host(ctype)
    if m and not name.endswith('_host') and m.group(1) in _DEVICE_DTYPES:
        return ctypes.c_void_p, _device(_DEVICE_DTYPES[m.group(1)])
    raise ImportError('%s: %s has a parameter "%s %s" of a type the binding does not know'
                      % (HEADER_PATH, function, c_type, name))


def _bind(function, restype, params):
    """-> (restype, argtypes, ((name, converter), ...), (the names a call must pass, with the optional ``stream``),
    whether it returns a status)."""
    if restype not in _RETURN_TYPES:
        raise ImportError('%s: %s returns a type the binding does not know: %s' % (HEADER_PATH, function, restype))
    typed = [_parameter(function, c_type, name) for c_type, name in params]
    names = frozenset(name for _, name in params)
    return (_RETURN_TYPES[restype], [argtype for argtype, _ in typed],
            tuple((name, convert) for (_, name), (_, convert) in zip(params, typed)),
            (names - {'stream'}, names), restype == 'int')


with open(HEADER_PATH) as _f:
    PROTOTYPES, _constants = parse_header(_f.read())
# PG_ERR_*, PG_ACT_*, PG_FLAG_*, PG_LAYER_*, PG_NMS_*, PG_KITTI_*, ... as the header defines them
globals().update(_constants)
KITTI_ROW_FIELDS = PG_KITTI_ROW_FIELDS  # noqa: F821
_BINDINGS = {function: _bind(function, *prototype) for function, prototype in PROTOTYPES.items()}
del _f, _constants

_lib = None
_FUNCTIONS = {}    # name -> the typed ctypes function, filled by load()


class PointGNNError(RuntimeError):
    """A C-ABI call returned a negative status."""

    def __init__(self, code, message):
        super().__init__('libpointgnn_b200 error %d: %s' % (code, message))
        self.code = code


def load():
    """Load (once) and type the shared library; raise if it is absent or incomplete."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.isfile(LIB_PATH):
        raise ImportError(
            'libpointgnn_b200.so not found at %s - build it with `python -c "import __graft_entry__ as g; '
            'g.build()"` or `make -C point-gnn_b200/csrc`; there is no CPU fallback' % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    for function, (restype, argtypes, _, _, _) in _BINDINGS.items():
        fn = getattr(lib, function)      # AttributeError if the symbol is missing
        fn.restype = restype
        fn.argtypes = argtypes
        _FUNCTIONS[function] = fn
    _lib = lib
    return lib


def _call(function, /, error=None, **args):
    """Call a PG_API function with its arguments bound by the header's parameter names; ``stream`` defaults to the
    current torch stream.  A negative status raises ``error`` (a PointGNNError subclass) when it lists the code in
    its ``codes``, else PointGNNError.  -> the return value."""
    _, _, params, (required, accepted), returns_status = _BINDINGS[function]
    keys = args.keys()
    if keys != required and keys != accepted:
        raise TypeError('%s(): missing %s, unexpected %s' % (function, sorted(required - keys), sorted(keys - accepted)))
    values = [args.get(name) if convert is None else convert(args.get(name), name) for name, convert in params]
    result = (_FUNCTIONS.get(function) or getattr(load(), function))(*values)
    if returns_status and result < 0:
        raise (error if error is not None and result in error.codes else PointGNNError)(
            result, _lib.pg_last_error().decode())
    return result


def _act_code(activation):
    """A PG_ACT_* code, checked here: a code outside [0, PG_ACT_COUNT) would not survive the int32 argument intact."""
    code = int(activation)
    if not 0 <= code < PG_ACT_COUNT:
        raise PointGNNError(PG_ERR_INVALID_ARGUMENT, 'unknown activation code %d' % code)
    return code


def _activation_flags(activation):
    """The precision-word flag bits that select a PG_ACT_* activation."""
    return PG_FLAG_ACTIVATION | (_act_code(activation) << PG_ACT_SHIFT)


def launch_count():
    return _call('pg_launch_count')


def device_is_sm90():
    return bool(_call('pg_device_is_sm90'))


def tc_launch_count(which=0):
    """tensor-core launches so far: which=0 segment-max (edge layer) launches, 1 dense-layer launches."""
    return _call('pg_tc_launch_count', which=int(which))


def tc_available():
    """True when the wgmma (precision=1 and 2) kernels are compiled in and the device is sm_90."""
    return bool(_call('pg_tc_available'))


# ---------------------------------------------------------------------------------------------
# graph construction
# ---------------------------------------------------------------------------------------------

def voxel_keypoints(xyz, frame_ptr, voxel_size):
    """-> (keypoint_idx [K] int32 global point rows, kp_frame_ptr [F+1] int32)."""
    n = xyz.shape[0]
    num_frames = frame_ptr.numel() - 1
    out_idx = torch.empty(n, dtype=torch.int32, device=xyz.device)
    out_fp = torch.empty(num_frames + 1, dtype=torch.int32, device=xyz.device)
    vs = (ctypes.c_double * 3)(*[float(v) for v in voxel_size])
    k = c_i64(0)
    _call('pg_voxel_keypoints', xyz=xyz, frame_ptr=frame_ptr, num_frames=num_frames, num_points=n, voxel_size_host=vs,
          out_keypoint_idx=out_idx, capacity=n, out_kp_frame_ptr=out_fp, out_num_keypoints_host=ctypes.byref(k))
    return out_idx[:k.value], out_fp


def voxel_centroids(xyz, frame_ptr, voxel_size):
    """pg_voxel_centroids -> (centroids [K,3] float64, frame_ptr [F+1] int32)."""
    n = xyz.shape[0]
    num_frames = frame_ptr.numel() - 1
    out = torch.empty((n, 3), dtype=torch.float64, device=xyz.device)
    out_fp = torch.empty(num_frames + 1, dtype=torch.int32, device=xyz.device)
    vs = (ctypes.c_double * 3)(*[float(v) for v in voxel_size])
    k = c_i64(0)
    _call('pg_voxel_centroids', xyz=xyz, frame_ptr=frame_ptr, num_frames=num_frames, num_points=n, voxel_size_host=vs,
          out_centroids=out, capacity=n, out_frame_ptr=out_fp, out_num_host=ctypes.byref(k))
    return out[:k.value], out_fp


def voxel_keypoints_select(xyz, frame_ptr, voxel_size, base_xyz, base_frame_ptr):
    """pg_voxel_keypoints_select -> (keypoint_idx [K] int32 rows of base_xyz, kp_frame_ptr [F+1] int32)."""
    n = xyz.shape[0]
    num_frames = frame_ptr.numel() - 1
    out_idx = torch.empty(n, dtype=torch.int32, device=xyz.device)
    out_fp = torch.empty(num_frames + 1, dtype=torch.int32, device=xyz.device)
    vs = (ctypes.c_double * 3)(*[float(v) for v in voxel_size])
    k = c_i64(0)
    _call('pg_voxel_keypoints_select', xyz=xyz, frame_ptr=frame_ptr, num_frames=num_frames, num_points=n,
          voxel_size_host=vs, base_xyz=base_xyz, base_frame_ptr=base_frame_ptr, num_base=base_xyz.shape[0],
          out_keypoint_idx=out_idx, capacity=n, out_kp_frame_ptr=out_fp, out_num_keypoints_host=ctypes.byref(k))
    return out_idx[:k.value], out_fp


def voxel_keypoints_rnd3d(xyz, frame_ptr, voxel_size, shift, base_xyz=None, base_frame_ptr=None, want_centroids=False):
    """pg_voxel_keypoints_rnd3d.  shift: [F,3] float64 host array.  -> (keypoint_idx [K] int32 rows of base_xyz or None,
    kp_frame_ptr [F+1] int32, centroids [K,3] float64 or None)."""
    n = xyz.shape[0]
    num_frames = frame_ptr.numel() - 1
    out_idx = torch.empty(n, dtype=torch.int32, device=xyz.device) if base_xyz is not None else None
    cent = torch.empty((n, 3), dtype=torch.float64, device=xyz.device) if want_centroids else None
    out_fp = torch.empty(num_frames + 1, dtype=torch.int32, device=xyz.device)
    vs = (ctypes.c_double * 3)(*[float(v) for v in voxel_size])
    k = c_i64(0)
    _call('pg_voxel_keypoints_rnd3d', xyz=xyz, frame_ptr=frame_ptr, num_frames=num_frames, num_points=n,
          voxel_size_host=vs, shift_host=np.ascontiguousarray(shift, dtype=np.float64).reshape(num_frames, 3),
          base_xyz=base_xyz, base_frame_ptr=base_frame_ptr, num_base=0 if base_xyz is None else base_xyz.shape[0],
          out_keypoint_idx=out_idx, out_centroids=cent, capacity=n, out_kp_frame_ptr=out_fp,
          out_num_keypoints_host=ctypes.byref(k))
    return (None if out_idx is None else out_idx[:k.value]), out_fp, (None if cent is None else cent[:k.value])


def random_keypoints(xyz, frame_ptr, voxel_size, shift, uniform):
    """pg_random_keypoints.  shift: None or [F,3] float64 host array; uniform: [N] CUDA fp32 in [0,1).
    -> (keypoint_idx [K] int32, kp_frame_ptr [F+1] int32)."""
    n = xyz.shape[0]
    num_frames = frame_ptr.numel() - 1
    out_idx = torch.empty(n, dtype=torch.int32, device=xyz.device)
    out_fp = torch.empty(num_frames + 1, dtype=torch.int32, device=xyz.device)
    vs = (ctypes.c_double * 3)(*[float(v) for v in voxel_size])
    sh = None if shift is None else np.ascontiguousarray(shift, dtype=np.float64).reshape(num_frames, 3)
    k = c_i64(0)
    _call('pg_random_keypoints', xyz=xyz, frame_ptr=frame_ptr, num_frames=num_frames, num_points=n,
          voxel_size_host=vs, shift_host=sh, uniform=uniform, out_keypoint_idx=out_idx, capacity=n,
          out_kp_frame_ptr=out_fp, out_num_keypoints_host=ctypes.byref(k))
    return out_idx[:k.value], out_fp


def cap_neighbors(row_ptr, edges, num_neighbors, seed):
    """pg_cap_neighbors on the (row_ptr, [2,E] edges) pair of radius_graph.  -> (row_ptr', [2,E'] edges)."""
    num_rows = row_ptr.numel() - 1
    e = edges.shape[1]
    out_rp = torch.empty_like(row_ptr)
    buf = torch.empty((2, max(e, 1)), dtype=torch.int32, device=edges.device)
    n = c_i64(0)
    src = edges[0].contiguous() if e else edges.new_zeros(1)
    _call('pg_cap_neighbors', row_ptr=row_ptr, src=src, num_rows=num_rows, num_neighbors=int(num_neighbors),
          seed=int(seed) & 0xffffffff, out_row_ptr=out_rp, out_src=buf[0], out_dst=buf[1], capacity=buf.shape[1],
          out_num_edges_host=ctypes.byref(n))
    return out_rp, buf[:, :n.value]


_edge_capacity = {}


def radius_graph(points, point_frame_ptr, centers, center_frame_ptr, radius, scale=None):
    """-> (row_ptr [K+1] int32, edges [2,E] int32 with row 0 = src, row 1 = dst).  scale: None or 3 positive
    per-axis divisors (graph_gen.py:203-206, float64 division inside the kernels)."""
    sc = None if scale is None else (ctypes.c_double * 3)(*[float(v) for v in scale])
    p, k = points.shape[0], centers.shape[0]
    num_frames = point_frame_ptr.numel() - 1
    row_ptr = torch.empty(k + 1, dtype=torch.int32, device=points.device)
    key = (points.device.index, float(radius), None if scale is None else tuple(float(v) for v in scale))
    cap = max(_edge_capacity.get(key, 0), 64 * k, 1 << 16)
    e = c_i64(0)
    while True:
        buf = torch.empty((2, cap), dtype=torch.int32, device=points.device)
        try:
            _call('pg_radius_graph_scaled', points=points, point_frame_ptr=point_frame_ptr, centers=centers,
                  center_frame_ptr=center_frame_ptr, num_frames=num_frames, num_points=p, num_centers=k,
                  radius=float(radius), scale_host=sc, out_row_ptr=row_ptr, out_src=buf[0], out_dst=buf[1],
                  capacity=cap, out_num_edges_host=ctypes.byref(e))
            break
        except PointGNNError as err:
            if err.code != PG_ERR_CAPACITY:
                raise
        cap = int(e.value * 1.25) + 1024
    _edge_capacity[key] = max(_edge_capacity.get(key, 0), int(e.value * 1.25) + 1024)
    # rows of buf are src / dst; the [E,2] transpose view of this slice has contiguous columns
    return row_ptr, buf[:, :e.value]


_graph_capacity = {}


def multi_level_graph(xyz, frame_ptr, voxel_size, radius0, radius1):
    """pg_multi_level_graph: keypoints + both radius graphs in one call with one host round trip.
    -> (kp_idx [K] int32, kp_frame_ptr [F+1] int32, kp_xyz [K,3], edges0 [2,E0], edges1 [2,E1])."""
    n = xyz.shape[0]
    num_frames = frame_ptr.numel() - 1
    dev = xyz.device
    key = (dev.index, int(n), tuple(float(v) for v in voxel_size), float(radius0), float(radius1))
    # buffer sizes: 1.25 x the largest result seen for this problem shape (first call: generous guesses)
    kcap, cap0, cap1 = _graph_capacity.get(key, (min(n, max(4096, n // 4)), 32 * n, 48 * n))
    vs = (ctypes.c_double * 3)(*[float(v) for v in voxel_size])
    sizes = (c_i64 * 3)()
    while True:
        kcap = min(int(kcap), n)
        kp_idx = torch.empty(kcap, dtype=torch.int32, device=dev)
        kp_fp = torch.empty(num_frames + 1, dtype=torch.int32, device=dev)
        kp_xyz = torch.empty((kcap, 3), dtype=torch.float32, device=dev)
        rp0 = torch.empty(kcap + 1, dtype=torch.int32, device=dev)
        rp1 = torch.empty(kcap + 1, dtype=torch.int32, device=dev)
        e0 = torch.empty((2, int(cap0)), dtype=torch.int32, device=dev)
        e1 = torch.empty((2, int(cap1)), dtype=torch.int32, device=dev)
        try:
            _call('pg_multi_level_graph', xyz=xyz, frame_ptr=frame_ptr, num_frames=num_frames, num_points=n,
                  voxel_size_host=vs, radius0=float(radius0), radius1=float(radius1), out_keypoint_idx=kp_idx,
                  kp_capacity=kcap, out_kp_frame_ptr=kp_fp, out_kp_xyz=kp_xyz, out_row_ptr0=rp0, out_src0=e0[0],
                  out_dst0=e0[1], capacity0=int(cap0), out_row_ptr1=rp1, out_src1=e1[0], out_dst1=e1[1],
                  capacity1=int(cap1), out_sizes_host=sizes)
            full = False
        except PointGNNError as err:
            if err.code != PG_ERR_CAPACITY:
                raise
            full = True
        k, n0, n1 = int(sizes[0]), int(sizes[1]), int(sizes[2])
        if not full:
            break
        if k > kcap:      # the edge counts were computed on a truncated keypoint set: scale them up too
            cap0, cap1 = max(cap0, int(n0 * 1.3 * k / kcap) + 1024), max(cap1, int(n1 * 1.7 * k / kcap) + 1024)
            kcap = int(k * 1.25) + 64
        elif n0 > cap0 or n1 > cap1:
            cap0, cap1 = max(cap0, int(n0 * 1.25) + 1024), max(cap1, int(n1 * 1.25) + 1024)
        else:             # the internal hit-parking buffer (10 x the edge capacity) overflowed
            cap0, cap1 = 2 * int(cap0), 2 * int(cap1)
    old = _graph_capacity.get(key, (0, 0, 0))
    _graph_capacity[key] = (max(old[0], int(k * 1.25) + 64), max(old[1], int(n0 * 1.25) + 1024),
                            max(old[2], int(n1 * 1.25) + 1024))
    return kp_idx[:k], kp_fp, kp_xyz[:k], e0[:, :n0], e1[:, :n1]


def radius_graph_two_pass(points, point_frame_ptr, centers, center_frame_ptr, radius):
    """The count / fill pair of the ABI (caller-allocated exact edge buffer)."""
    k = centers.shape[0]
    row_ptr = torch.empty(k + 1, dtype=torch.int32, device=points.device)
    e = c_i64(0)
    args = dict(points=points, point_frame_ptr=point_frame_ptr, centers=centers, center_frame_ptr=center_frame_ptr,
                num_frames=point_frame_ptr.numel() - 1, num_points=points.shape[0], num_centers=k,
                radius=float(radius))
    _call('pg_radius_graph_count', **args, out_row_ptr=row_ptr, out_num_edges_host=ctypes.byref(e))
    out = torch.empty((2, e.value), dtype=torch.int32, device=points.device)
    _call('pg_radius_graph_fill', **args, row_ptr=row_ptr, num_edges=e.value, out_src=out[0], out_dst=out[1])
    return row_ptr, out


# ---------------------------------------------------------------------------------------------
# GNN ops
# ---------------------------------------------------------------------------------------------

def scatter_max(features, centers, num_centers):
    e, c = features.shape
    out = torch.empty((int(num_centers), c), dtype=torch.float32, device=features.device)
    _call('pg_scatter_max', features=features, centers=centers, num_edges=e, num_channels=c,
          num_centers=int(num_centers), out=out)
    return out


def scatter_sum(features, centers, num_centers, mean=False):
    e, c = features.shape
    out = torch.empty((int(num_centers), c), dtype=torch.float32, device=features.device)
    _call('pg_scatter_mean' if mean else 'pg_scatter_sum', features=features, centers=centers, num_edges=e,
          num_channels=c, num_centers=int(num_centers), out=out)
    return out


def gather_rows(params, indices):
    r, c = params.shape
    n = indices.numel()
    out = torch.empty((n, c), dtype=torch.float32, device=params.device)
    _call('pg_gather_rows', params=params, num_rows=r, num_channels=c, indices=indices, num_indices=n, out=out)
    return out


def _check_fc_shapes(x, k, n, residual):
    """x [m, k] into a layer chain of input width k and output width n; the optional residual must be [m, n]."""
    m = x.shape[0]
    if x.shape[1] != k:
        raise ValueError('fully_connected: input width %d != weight rows %d' % (x.shape[1], k))
    if residual is not None and tuple(residual.shape) != (m, n):
        # the reference's tf add raises a shape error here (gnn.py:346, 372)
        raise ValueError('fully_connected: residual shape %s != output shape (%d, %d)' % (tuple(residual.shape), m, n))


def fully_connected(x, w, b, relu, residual=None, precision=0, activation=None):
    """activation: a PG_ACT_* code; None = ReLU or linear as ``relu`` says."""
    if activation is None:
        activation = PG_ACT_RELU if relu else PG_ACT_NONE
    m, k = x.shape
    n = w.shape[1]
    _check_fc_shapes(x, w.shape[0], n, residual)
    if b.numel() != n:
        raise ValueError('fully_connected: bias has %d entries, layer width is %d' % (b.numel(), n))
    out = torch.empty((m, n), dtype=torch.float32, device=x.device)
    _call('pg_fully_connected', x=x, m=m, k=k, w=w, bias=b, n=n, act=_act_code(activation), residual=residual,
          out=out, precision=int(precision))
    return out


def check_edges(src, dst, num_src, num_dst):
    """Raise PointGNNError unless 0 <= src < num_src and 0 <= dst < num_dst (one synchronising kernel)."""
    _call('pg_check_edges', src=src, dst=dst, num_edges=src.numel(), num_src=int(num_src), num_dst=int(num_dst))


def edge_mlp_max(mode, features, xyz_src, xyz_dst, dst_index, src, dst, num_dst, weights, biases, precision=0,
                 trusted=False, activation=PG_ACT_RELU):
    """trusted=True: the caller vouches for the index ranges (graph_gen output / check_edges passed); the call
    then does not read the range-error flag back and does not synchronise the stream.  activation: the PG_ACT_* code
    applied after every layer."""
    num_layers = len(weights)
    dims = [weights[0].shape[0]] + [w.shape[1] for w in weights]
    out = torch.empty((int(num_dst), dims[-1]), dtype=torch.float32, device=features.device)
    _call('pg_edge_mlp_max', mode=int(mode), features=features, num_feature_channels=features.shape[1],
          xyz_src=xyz_src, xyz_dst=xyz_dst, dst_index=dst_index, src=src, dst=dst, num_edges=src.numel(),
          num_src=features.shape[0], num_dst=int(num_dst), weights_host=weights, biases_host=biases,
          dims_host=(c_i32 * (num_layers + 1))(*dims), num_layers=num_layers, out=out,
          precision=int(precision) | (PG_FLAG_TRUSTED_INDICES if trusted else 0) | _activation_flags(activation))
    return out


def softmax_rows(logits):
    out = torch.empty_like(logits)
    _call('pg_softmax_rows', logits=logits, num_rows=logits.shape[0], num_classes=logits.shape[1], out=out)
    return out


# ---------------------------------------------------------------------------------------------
# prepared layers (weights packed once; the calls below launch compute kernels only)
# ---------------------------------------------------------------------------------------------
class PreparedLayer(object):
    """Owner of one ``pg_layer`` handle.  Keeps the weight tensors alive: the C side stores their pointers."""

    def __init__(self, kind, weights, biases, dims, precision=0, activation=PG_ACT_RELU):
        """activation: the PG_ACT_* code of every layer that has one (the is_logits last layers stay linear)."""
        self.kind = int(kind)
        self.activation = int(activation)
        self.dims = [int(d) for d in dims]
        self._keep = (list(weights), list(biases))
        handle = ctypes.c_void_p()
        self._handle = None
        _call('pg_layer_create', kind=self.kind, weights_host=self._keep[0], biases_host=self._keep[1],
              dims_host=(c_i32 * len(self.dims))(*self.dims), num_layers=len(self._keep[0]),
              precision=int(precision) | _activation_flags(activation), out_layer=ctypes.byref(handle))
        self._handle = handle

    def __del__(self):
        if getattr(self, '_handle', None) is not None and _lib is not None:
            _call('pg_layer_destroy', layer=self._handle)
            self._handle = None

    # multi_layer_neural_network_fn / multi_layer_fc_fn (gnn.py:34-104)
    def mlp(self, x, last_linear, residual=None):
        m, _ = x.shape
        n = self.dims[-1]
        _check_fc_shapes(x, self.dims[0], n, residual)
        out = torch.empty((m, n), dtype=torch.float32, device=x.device)
        _call('pg_layer_mlp', layer=self._handle, x=x, m=m, last_linear=1 if last_linear else 0, residual=residual,
              out=out)
        return out

    # fused gather -> edge MLP -> segment max (gnn.py:256-277, 338-365)
    def edge_mlp_max(self, features, xyz_src, xyz_dst, dst_index, src, dst, num_dst, trusted=False):
        if features.shape[1] + 3 != self.dims[0]:
            raise ValueError('edge layer: %d feature channels + 3 != first weight rows %d'
                             % (features.shape[1], self.dims[0]))
        out = torch.empty((int(num_dst), self.dims[-1]), dtype=torch.float32, device=features.device)
        _call('pg_layer_edge_mlp_max', layer=self._handle, features=features, xyz_src=xyz_src, xyz_dst=xyz_dst,
              dst_index=dst_index, src=src, dst=dst, num_edges=src.numel(), num_src=features.shape[0],
              num_dst=int(num_dst), out=out, flags=PG_FLAG_TRUSTED_INDICES if trusted else 0)
        return out

    # ClassAwarePredictor (gnn.py:133-163) + softmax (models.py:165-168)
    def predictor(self, x):
        d, h, c, box = self.dims
        m = x.shape[0]
        if x.shape[1] != d:
            raise ValueError('predictor: input width %d != %d' % (x.shape[1], d))
        logits = torch.empty((m, c), dtype=torch.float32, device=x.device)
        probs = torch.empty((m, c), dtype=torch.float32, device=x.device)
        boxes = torch.empty((m, c, box), dtype=torch.float32, device=x.device)
        _call('pg_layer_predictor', layer=self._handle, x=x, m=m, logits=logits, boxes=boxes, probs=probs)
        return logits, boxes, probs


# ---------------------------------------------------------------------------------------------
# post-processing (box decoding + NMS)
# ---------------------------------------------------------------------------------------------
MAX_CANDIDATES_PER_FRAME = 16384


def _class_table(table):
    flat = [float(v) for row in table for v in row]
    return (ctypes.c_float * len(flat))(*flat)


def decode_boxes(box_encodings, xyz, class_table):
    """[K, C, 7] encodings at the K vertices -> [K, C, 7] boxes (box_encoding.py:265-299)."""
    k, c, _ = box_encodings.shape
    out = torch.empty_like(box_encodings)
    _call('pg_decode_boxes', box_encodings=box_encodings, xyz=xyz, num_vertices=k, num_classes=c,
          class_table_host=_class_table(class_table), out_boxes=out)
    return out


def postprocess(probs, box_encodings, xyz, frame_ptr, class_table, overlapped_thres, merge=True, rescore=True,
                want_candidates=False):
    """run.py:265-325 for a batch of frames on the device.
    -> dict(label [D] int32, box [D,7], score [D], index [D] int32, frame_ptr [F+1] int32
            [, cand_index [B] int32, cand_frame_ptr [F+1] int32])."""
    k, c = probs.shape
    num_frames = frame_ptr.numel() - 1
    dev = probs.device
    cap = max(1024, k)
    flags = (PG_NMS_MERGE if merge else 0) | (PG_NMS_RESCORE if rescore else 0)
    sizes = (c_i64 * 2)()
    cand_index = torch.empty(k * max(c - 2, 1), dtype=torch.int32, device=dev) if want_candidates else None
    cand_fp = torch.empty(num_frames + 1, dtype=torch.int32, device=dev) if want_candidates else None
    while True:
        label = torch.empty(cap, dtype=torch.int32, device=dev)
        box = torch.empty((cap, 7), dtype=torch.float32, device=dev)
        score = torch.empty(cap, dtype=torch.float32, device=dev)
        index = torch.empty(cap, dtype=torch.int32, device=dev)
        det_fp = torch.empty(num_frames + 1, dtype=torch.int32, device=dev)
        try:
            _call('pg_postprocess', probs=probs, box_encodings=box_encodings, xyz=xyz, frame_ptr=frame_ptr,
                  num_frames=num_frames, num_vertices=k, num_classes=c, class_table_host=_class_table(class_table),
                  overlapped_thres=float(overlapped_thres), flags=flags,
                  max_candidates_per_frame=MAX_CANDIDATES_PER_FRAME, out_label=label, out_box=box, out_score=score,
                  out_index=index, capacity=cap, out_det_frame_ptr=det_fp, out_cand_index=cand_index,
                  out_cand_frame_ptr=cand_fp, out_sizes_host=sizes)
            break
        except PointGNNError as err:
            if err.code != PG_ERR_CAPACITY or int(sizes[0]) <= cap:
                raise
        cap = int(sizes[0])
    d, b = int(sizes[0]), int(sizes[1])
    out = dict(label=label[:d], box=box[:d], score=score[:d], index=index[:d], frame_ptr=det_fp)
    if want_candidates:
        out['cand_index'] = cand_index[:b]
        out['cand_frame_ptr'] = cand_fp
    return out


def nms_boxes_3d(class_labels, boxes, scores, frame_ptr, overlapped_thres, merge, rescore, appr_factor=0.0,
                 int_corners=False):
    """models/nms.py's entry points on caller-provided boxes.  -> (label, box, score, index, det_frame_ptr)."""
    n = boxes.shape[0]
    num_frames = frame_ptr.numel() - 1
    dev = boxes.device
    flags = (PG_NMS_MERGE if merge else 0) | (PG_NMS_RESCORE if rescore else 0) | (PG_NMS_INT_CORNERS if int_corners else 0)
    sizes = (c_i64 * 2)()
    label = torch.empty(n, dtype=torch.int32, device=dev)
    box = torch.empty((n, 7), dtype=torch.float32, device=dev)
    score = torch.empty(n, dtype=torch.float32, device=dev)
    index = torch.empty(n, dtype=torch.int32, device=dev)
    det_fp = torch.empty(num_frames + 1, dtype=torch.int32, device=dev)
    _call('pg_nms_boxes_3d', class_labels=class_labels, boxes=boxes, scores=scores, frame_ptr=frame_ptr,
          num_frames=num_frames, num_boxes=n, overlapped_thres=float(overlapped_thres), appr_factor=float(appr_factor),
          flags=flags, max_candidates_per_frame=MAX_CANDIDATES_PER_FRAME, out_label=label, out_box=box,
          out_score=score, out_index=index, capacity=n, out_det_frame_ptr=det_fp, out_sizes_host=sizes)
    d = int(sizes[0])
    return label[:d], box[:d], score[:d], index[:d], det_fp


def kitti_rows(label, box, score, det_frame_ptr, xyz, cand_index, cand_frame_ptr, num_classes, cam_to_image, rescore):
    """pg_kitti_rows.  The detections and candidates as ``postprocess`` returns them, xyz [K,3] the last-level
    vertices, cam_to_image [F,3,4] CUDA float64.  -> (rows [R, KITTI_ROW_FIELDS] float64, row_frame_ptr [F+1] int32),
    the row layout of include/pointgnn_b200.h."""
    num_frames = det_frame_ptr.numel() - 1
    d = box.shape[0]
    dev = box.device
    if tuple(cam_to_image.shape) != (num_frames, 3, 4):
        raise ValueError('cam_to_image must be [%d, 3, 4], got %s' % (num_frames, tuple(cam_to_image.shape)))
    rows = torch.empty((max(d, 1), KITTI_ROW_FIELDS), dtype=torch.float64, device=dev)
    row_fp = torch.empty(num_frames + 1, dtype=torch.int32, device=dev)
    n = c_i64(0)
    _call('pg_kitti_rows', boxes=box, labels=label, scores=score, det_frame_ptr=det_frame_ptr, num_frames=num_frames,
          num_dets=d, xyz=xyz, cand_index=cand_index, cand_frame_ptr=cand_frame_ptr, num_classes=int(num_classes),
          cam_to_image=cam_to_image, flags=PG_KITTI_ROWS_RESCORE if rescore else 0, out_rows=rows,
          out_row_frame_ptr=row_fp, out_num_rows_host=ctypes.byref(n))
    return rows[:n.value], row_fp


# ---------------------------------------------------------------------------------------------
# input stage
# ---------------------------------------------------------------------------------------------
def _crop_args(num_frames, cam_to_image, image_sizes, images, image_offsets):
    """The image arguments both crop entry points take, by name."""
    return dict(cam_to_image_host=np.ascontiguousarray(cam_to_image, dtype=np.float64).reshape(num_frames, 12),
                image_size_host=np.ascontiguousarray(image_sizes, dtype=np.int32).reshape(num_frames, 2),
                images=images,
                image_offset_host=None if images is None else np.ascontiguousarray(image_offsets, dtype=np.int64))


def cam_points_in_image(velo, frame_ptr, velo_to_cam, cam_to_image, image_sizes, images=None, image_offsets=None):
    """pg_cam_points_in_image.  velo [M,4] CUDA fp32, frame_ptr [F+1] CUDA int32, velo_to_cam [F,4,4] / cam_to_image
    [F,3,4] / image_sizes [F,2] host arrays; images: optional CUDA uint8 buffer (+ byte offsets per frame).
    -> (xyz [N,3], attr [N,1 or 4], out_frame_ptr [F+1])."""
    m = velo.shape[0]
    num_frames = frame_ptr.numel() - 1
    channels = 4 if images is not None else 1
    out_xyz = torch.empty((m, 3), dtype=torch.float32, device=velo.device)
    out_attr = torch.empty((m, channels), dtype=torch.float32, device=velo.device)
    out_fp = torch.empty(num_frames + 1, dtype=torch.int32, device=velo.device)
    n = c_i64(0)
    _call('pg_cam_points_in_image', velo_points=velo, frame_ptr=frame_ptr, num_frames=num_frames, num_points=m,
          velo_to_cam_host=np.ascontiguousarray(velo_to_cam, dtype=np.float32).reshape(num_frames, 16),
          **_crop_args(num_frames, cam_to_image, image_sizes, images, image_offsets), out_xyz=out_xyz,
          out_attr=out_attr, attr_channels=channels, capacity=m, out_frame_ptr=out_fp,
          out_num_points_host=ctypes.byref(n))
    return out_xyz[:n.value], out_attr[:n.value], out_fp


def velo_to_cam(velo, frame_ptr, velo_to_cam):
    """pg_velo_to_cam: the transform of ``cam_points_in_image`` alone, same argument forms.
    -> (xyz [M,3] camera-frame points, attr [M,1] reflectance)."""
    m = velo.shape[0]
    num_frames = frame_ptr.numel() - 1
    out_xyz = torch.empty((m, 3), dtype=torch.float32, device=velo.device)
    out_attr = torch.empty((m, 1), dtype=torch.float32, device=velo.device)
    _call('pg_velo_to_cam', velo_points=velo, frame_ptr=frame_ptr, num_frames=num_frames, num_points=m,
          velo_to_cam_host=np.ascontiguousarray(velo_to_cam, dtype=np.float32).reshape(num_frames, 16),
          out_xyz=out_xyz, out_attr=out_attr)
    return out_xyz, out_attr


def cam_points_crop(xyz, reflectance, frame_ptr, cam_to_image, image_sizes, images=None, image_offsets=None):
    """pg_cam_points_crop: the crop and colour lookup of ``cam_points_in_image`` from camera-frame points xyz [N,3] with
    reflectance [N,1] (CUDA fp32).  The other arguments and the result are ``cam_points_in_image``'s."""
    n_in = xyz.shape[0]
    num_frames = frame_ptr.numel() - 1
    channels = 4 if images is not None else 1
    out_xyz = torch.empty((n_in, 3), dtype=torch.float32, device=xyz.device)
    out_attr = torch.empty((n_in, channels), dtype=torch.float32, device=xyz.device)
    out_fp = torch.empty(num_frames + 1, dtype=torch.int32, device=xyz.device)
    n = c_i64(0)
    _call('pg_cam_points_crop', cam_xyz=xyz, reflectance=reflectance, frame_ptr=frame_ptr, num_frames=num_frames,
          num_points=n_in, **_crop_args(num_frames, cam_to_image, image_sizes, images, image_offsets),
          out_xyz=out_xyz, out_attr=out_attr, attr_channels=channels, capacity=n_in, out_frame_ptr=out_fp,
          out_num_points_host=ctypes.byref(n))
    return out_xyz[:n.value], out_attr[:n.value], out_fp


class VoxelAverageError(PointGNNError, ValueError):
    """pg_voxel_average rejected the voxel size, or a frame has more voxels than the reference's int32 voxel key (or
    the grid's 16 bits per axis) can number."""
    codes = (PG_ERR_INVALID_ARGUMENT, PG_ERR_RANGE)


def voxel_average(xyz, attr, frame_ptr, voxel_size):
    """pg_voxel_average.  xyz [M,3] CUDA fp32, attr None or [M,C] CUDA fp32 with C <= 4, frame_ptr [F+1] CUDA int32.
    -> (xyz [V,3], attr [V,C] or None, frame_ptr [F+1]): one point per occupied voxel, see include/pointgnn_b200.h."""
    import math
    voxel_size = float(voxel_size)
    if not (voxel_size > 0.0 and math.isfinite(voxel_size)):
        raise VoxelAverageError(PG_ERR_INVALID_ARGUMENT, 'voxel_size must be positive and finite, got %r' % voxel_size)
    if xyz.dim() != 2 or xyz.shape[1] != 3:
        raise ValueError('xyz must be [M, 3], got %s' % (tuple(xyz.shape),))
    m = xyz.shape[0]
    if attr is not None and (attr.dim() != 2 or attr.shape[0] != m):
        raise ValueError('attr must be [%d, C], got %s' % (m, tuple(attr.shape)))
    channels = 0 if attr is None else attr.shape[1]
    num_frames = frame_ptr.numel() - 1
    out_xyz = torch.empty((m, 3), dtype=torch.float32, device=xyz.device)
    out_attr = None if attr is None else torch.empty((m, channels), dtype=torch.float32, device=xyz.device)
    out_fp = torch.empty(num_frames + 1, dtype=torch.int32, device=xyz.device)
    n = c_i64(0)
    _call('pg_voxel_average', error=VoxelAverageError, xyz=xyz, attr=attr, attr_channels=channels, frame_ptr=frame_ptr,
          num_frames=num_frames, num_points=m, voxel_size=voxel_size, out_xyz=out_xyz, out_attr=out_attr, capacity=m,
          out_frame_ptr=out_fp, out_num_host=ctypes.byref(n))
    return out_xyz[:n.value], None if attr is None else out_attr[:n.value], out_fp


# ---------------------------------------------------------------------------------------------
# LiDAR beam downsampling
# ---------------------------------------------------------------------------------------------
class BeamDownsampleError(PointGNNError, ValueError):
    """pg_beam_downsample rejected its arguments (a frame with fewer finite cosines than clusters, or a bad rate /
    cluster count), as scikit-learn's KMeans raises ValueError."""
    codes = (PG_ERR_INVALID_ARGUMENT,)


def beam_downsample(velo, frame_ptr, num_clusters, downsample_rate, centers_in=None):
    """pg_beam_downsample.  velo [M,4] CUDA float32, frame_ptr [F+1] CUDA int32; centers_in: None (exact 1-D k-means per
    frame) or [F, num_clusters] CUDA float64.  -> dict(velo [R,4] float32 kept rows, frame_ptr [F+1] int32,
    centers [F,K] float64, and without centers_in: inertia [F] float64, group_sizes [F,K] int32)."""
    num_frames = frame_ptr.numel() - 1
    k, rate = int(num_clusters), int(downsample_rate)
    if k < 1 or rate < 1:
        raise BeamDownsampleError(PG_ERR_INVALID_ARGUMENT, 'num_clusters and downsample_rate must be >= 1, got %d and %d'
                                  % (k, rate))
    if velo.dim() != 2 or velo.shape[1] != 4:
        raise ValueError('velo must be [M, 4], got %s' % (tuple(velo.shape),))
    m = velo.shape[0]
    dev = velo.device
    if centers_in is not None and tuple(centers_in.shape) != (num_frames, k):
        raise ValueError('centers_in must be [%d, %d], got %s' % (num_frames, k, tuple(centers_in.shape)))
    if centers_in is not None:   # the script sorts the centres it is given (point_cloud_downsample.py:27)
        centers_in = torch.sort(centers_in, dim=1).values.contiguous()
    centers =torch.empty((num_frames, k), dtype=torch.float64, device=dev)
    inertia = torch.empty(num_frames, dtype=torch.float64, device=dev) if centers_in is None else None
    sizes = torch.empty((num_frames, k), dtype=torch.int32, device=dev) if centers_in is None else None
    out = torch.empty((max(m, 1), 4), dtype=torch.float32, device=dev)
    out_fp = torch.empty(num_frames + 1, dtype=torch.int32, device=dev)
    n = c_i64(0)
    _call('pg_beam_downsample', error=BeamDownsampleError, velo=velo, frame_ptr=frame_ptr, num_frames=num_frames,
          num_points=m, num_clusters=k, downsample_rate=rate, centers_in=centers_in, centers_out=centers,
          inertia_out=inertia, group_sizes_out=sizes, out_velo=out, out_frame_ptr=out_fp,
          out_num_points_host=ctypes.byref(n))
    res = dict(velo=out[:n.value], frame_ptr=out_fp, centers=centers)
    if centers_in is None:
        res.update(inertia=inertia, group_sizes=sizes)
    return res


# ---------------------------------------------------------------------------------------------
# KITTI object evaluation
# ---------------------------------------------------------------------------------------------
def kitti_eval(gt, gt_class, det, det_class, gt_frame_ptr, det_frame_ptr, compute_aos):
    """pg_kitti_eval.  gt [G,14] / det [D,15] CUDA float64, gt_class / det_class CUDA int32, frame pointers [F+1] host
    int64 arrays.  -> dict of host arrays: precision / aos / ahs [3,3,3,41] float64, num_thresholds [3,3,3],
    tp / fp / fn [3,3,3,41] int32 (axes: metric, class, difficulty, threshold)."""
    gfp = np.ascontiguousarray(gt_frame_ptr, dtype=np.int64)
    dfp = np.ascontiguousarray(det_frame_ptr, dtype=np.int64)
    out = {k: np.zeros((3, 3, 3, 41), np.float64) for k in ('precision', 'aos', 'ahs')}
    out.update({k: np.zeros((3, 3, 3, 41), np.int32) for k in ('tp', 'fp', 'fn')})
    out['num_thresholds'] = np.zeros((3, 3, 3), np.int32)
    _call('pg_kitti_eval', gt=gt, gt_class=gt_class, det=det, det_class=det_class, gt_frame_ptr_host=gfp,
          det_frame_ptr_host=dfp, num_frames=len(gfp) - 1, flags=PG_KITTI_EVAL_AOS if compute_aos else 0,
          out_precision_host=out['precision'], out_aos_host=out['aos'], out_ahs_host=out['ahs'],
          out_num_thresholds_host=out['num_thresholds'], out_tp_host=out['tp'], out_fp_host=out['fp'],
          out_fn_host=out['fn'])
    return out
