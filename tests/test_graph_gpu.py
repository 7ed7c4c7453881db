"""GPU parity tests for graph construction: CUDA kernels (through the C ABI) vs the CPU oracle
and vs the golden edge lists produced by the reference's own graph_gen.py.  Bit-exact."""
import numpy as np
import pytest
import torch

from oracle import graph, synth

pytestmark = pytest.mark.gpu


def _np(t):
    return t.cpu().numpy()


def _check_graph(xyz, kwargs, got):
    coords_o, kp_o, edges_o = graph.gen_multi_level_local_graph_v3(xyz, **kwargs)
    coords, kp, edges = got
    assert len(coords) == len(coords_o) and len(edges) == len(edges_o)
    for a, b in zip(coords, coords_o):
        assert np.array_equal(np.asarray(a), np.asarray(b, dtype=np.float32))
    for a, b in zip(kp, kp_o):
        assert a.shape == b.shape and np.array_equal(a, b)
    for a, b in zip(edges, edges_o):
        assert a.shape == b.shape and np.array_equal(a, b)      # already canonical: no re-sort needed


@pytest.mark.parametrize('name', ['car', 'ped'])
def test_numpy_api_matches_reference_golden(name, request):
    from pointgnn_b200.models import graph_gen
    g = request.getfixturevalue(name)
    fn = graph_gen.get_graph_generate_fn(g.config['graph_gen_method'])
    coords, kp, edges = fn(g.graph['xyz'], **g.graph_kwargs)
    assert isinstance(edges[0], np.ndarray) and edges[0].dtype == np.int64 and edges[0].shape[1] == 2
    assert np.array_equal(kp[0][:, 0], g.graph['keypoint_idx'])
    assert np.array_equal(edges[0], g.graph['edges0'])          # reference's sklearn output, canonical order
    assert np.array_equal(edges[1], g.graph['edges1'])
    assert np.array_equal(coords[1], g.graph['xyz'][g.graph['keypoint_idx']])


@pytest.mark.parametrize('n,frame', [(20000, 0), (6000, 3)])
def test_full_frame_vs_oracle(car, n, frame):
    from pointgnn_b200.models import graph_gen
    xyz, _ = synth.lidar_frame(frame, n)
    got = graph_gen.gen_multi_level_local_graph_v3(xyz, **car.graph_kwargs)
    _check_graph(xyz, car.graph_kwargs, got)


def test_ped_radii_vs_oracle(ped):
    from pointgnn_b200.models import graph_gen
    xyz, _ = synth.lidar_frame(2, 12000)
    got = graph_gen.gen_multi_level_local_graph_v3(xyz, **ped.graph_kwargs)
    _check_graph(xyz, ped.graph_kwargs, got)


def test_device_tensor_api_and_two_pass_abi(car):
    from pointgnn_b200 import _lib
    from pointgnn_b200.models import graph_gen
    xyz, _ = synth.lidar_frame(4, 5000)
    t = torch.from_numpy(xyz).cuda()
    coords, kp, edges = graph_gen.gen_multi_level_local_graph_v3(t, **car.graph_kwargs)
    assert all(c.is_cuda for c in coords) and edges[0].is_cuda and edges[0].dtype == torch.int32
    assert edges[0][:, 0].is_contiguous() and edges[0][:, 1].is_contiguous()
    _check_graph(xyz, car.graph_kwargs, ([_np(c) for c in coords], [_np(k).astype(np.int64) for k in kp],
                                        [_np(e).astype(np.int64) for e in edges]))
    fp = torch.tensor([0, 5000], dtype=torch.int32, device='cuda')
    kfp = torch.tensor([0, coords[1].shape[0]], dtype=torch.int32, device='cuda')
    row_ptr, e2 = _lib.radius_graph_two_pass(t, fp, coords[1], kfp, 1.0)
    assert np.array_equal(_np(e2.t()), _np(edges[0]))
    rp = _np(row_ptr)
    assert rp[0] == 0 and rp[-1] == e2.shape[1]
    assert np.array_equal(np.diff(rp), np.bincount(_np(e2[1]), minlength=coords[1].shape[0]))


def test_batched_frames_equal_batch_data(car):
    """frame_ptr batching == reference batch_data (train.py:135-171) of per-frame graphs."""
    from pointgnn_b200.models import graph_gen
    clouds = [synth.lidar_frame(i, n)[0] for i, n in ((20, 3000), (21, 4500), (22, 2000))]
    frames = []
    for c in clouds:
        co, kp, ed = graph.gen_multi_level_local_graph_v3(c, **car.graph_kwargs)
        frames.append((np.zeros((c.shape[0], 1), np.float32), co, kp, ed))
    _, bc, bk, be = graph.batch_graphs(frames)
    fp = np.cumsum([0] + [c.shape[0] for c in clouds]).astype(np.int32)
    coords, kp, edges, fps = graph_gen.gen_multi_level_local_graph_v3(
        np.vstack(clouds), frame_ptr=fp, return_frame_ptr=True, **car.graph_kwargs)
    for a, b in zip(coords, bc):
        assert np.array_equal(a, b.astype(np.float32))
    for a, b in zip(kp, bk):
        assert np.array_equal(a, b)
    for a, b in zip(edges, be):
        assert np.array_equal(a, b)
    assert np.array_equal(fps[1], np.cumsum([0] + [f[1][1].shape[0] for f in frames]))


def test_edge_cases():
    from pointgnn_b200.models import graph_gen
    # single point: one keypoint, one self loop at every level
    one = np.array([[1.5, -0.25, 7.0]], np.float32)
    cfg = [dict(graph_level=0, graph_scale=0.5, graph_gen_method='disjointed_rnn_local_graph_v3',
                graph_gen_kwargs=dict(radius=1.0, num_neighbors=-1)),
           dict(graph_level=1, graph_scale=0.5, graph_gen_method='disjointed_rnn_local_graph_v3',
                graph_gen_kwargs=dict(radius=4.0, num_neighbors=-1))]
    coords, kp, edges = graph_gen.gen_multi_level_local_graph_v3(one, 0.8, cfg)
    assert np.array_equal(kp[0], [[0]]) and np.array_equal(edges[0], [[0, 0]]) and np.array_equal(edges[1], [[0, 0]])
    # exact boundary: points at distance exactly r are included (d <= r), just outside are not
    pts = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, np.nextafter(np.float32(1), np.float32(2))],
                    [0.6, 0.8, 0]], np.float32)
    e = graph_gen.gen_disjointed_rnn_local_graph_v3(pts, pts[:1], 1.0, -1)
    assert np.array_equal(e, graph.radius_graph(pts, pts[:1], 1.0))
    assert e[:, 0].tolist() == [0, 1, 2] or e[:, 0].tolist() == [0, 1, 2, 4]   # 0.36+0.64 rounds either way in fp32->fp64
    # dense blob: every point within the radius of every centre -> one very long row per centre
    rng = np.random.default_rng(0)
    blob = (rng.random((9000, 3), dtype=np.float32) * 0.3).astype(np.float32)
    e = graph_gen.gen_disjointed_rnn_local_graph_v3(blob, blob[:3], 1.0, -1)
    assert e.shape == (27000, 2) and np.array_equal(e, graph.radius_graph(blob, blob[:3], 1.0))
    # centres outside the bounding box of the points, negative coordinates, empty rows
    pts = (rng.random((500, 3), dtype=np.float32) * 10 - 5).astype(np.float32)
    ctr = np.array([[-30, 0, 0], [0, 0, 0], [4.9, 4.9, 4.9], [100, 100, 100]], np.float32)
    e = graph_gen.gen_disjointed_rnn_local_graph_v3(pts, ctr, 2.0, -1)
    assert np.array_equal(e, graph.radius_graph(pts, ctr, 2.0))
    # duplicate points: ties in the 1-NN snap resolve to the lowest index, duplicates are kept
    dup = np.repeat(np.array([[0.1, 0.1, 5.0], [3.0, 0.2, 9.0]], np.float32), 3, axis=0)
    coords, kp, edges = graph_gen.gen_multi_level_local_graph_v3(dup, 0.8, cfg)
    co, ko, eo = graph.gen_multi_level_local_graph_v3(dup, 0.8, cfg)
    assert np.array_equal(kp[0], ko[0]) and np.array_equal(edges[0], eo[0]) and np.array_equal(edges[1], eo[1])


def test_per_axis_voxel_and_training_paths_raise(car):
    from pointgnn_b200.models import graph_gen
    xyz, _ = synth.lidar_frame(9, 3000)
    kw = dict(car.graph_kwargs)
    kw['base_voxel_size'] = [0.8, 0.6, 1.0]                   # graph_gen.py:172-173
    got = graph_gen.gen_multi_level_local_graph_v3(xyz, **kw)
    _check_graph(xyz, kw, got)
    with pytest.raises(KeyError):
        graph_gen.gen_multi_level_local_graph_v3(xyz, 0.8, car.graph_kwargs['level_configs'], downsample_method='nope')


def test_large_cloud_properties(car):
    """120k-point 360-degree frame (BASELINE config 3): size-independent properties + oracle."""
    from pointgnn_b200.models import graph_gen
    xyz, _ = synth.lidar_frame(1, 120000, full_360=True)
    coords, kp, edges = graph_gen.gen_multi_level_local_graph_v3(xyz, **car.graph_kwargs)
    k = kp[0].shape[0]
    for e, nsrc in ((edges[0], xyz.shape[0]), (edges[1], k)):
        assert np.all(np.diff(e[:, 1]) >= 0)
        same = e[1:, 1] == e[:-1, 1]
        assert np.all(e[1:, 0][same] > e[:-1, 0][same])
        assert e[:, 0].min() >= 0 and e[:, 0].max() < nsrc and e[:, 1].max() == k - 1
    e1 = edges[1]
    assert np.count_nonzero(e1[:, 0] == e1[:, 1]) == k                        # self loops
    # symmetry of the keypoint graph: (a,b) in E <=> (b,a) in E
    fwd = e1[:, 0] * k + e1[:, 1]
    bwd = e1[:, 1] * k + e1[:, 0]
    assert np.array_equal(np.sort(fwd), np.sort(bwd))
    _check_graph(xyz, car.graph_kwargs, (coords, kp, edges))


def test_multiscale_downsampling_vs_reference_golden():
    """General multi-scale keypoint selection (a second and third distinct scale: the voxel centroids of the ORIGINAL
    cloud snapped to the nearest vertex of the PREVIOUS level, graph_gen.py:17-23, 41-45, 76-88) against the
    reference's own multi_layer_downsampling_select / multi_layer_downsampling (tests/golden/graph_multiscale.npz)."""
    import os
    from pointgnn_b200.models import graph_gen
    g = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'graph_multiscale.npz'))
    levels = [float(v) for v in g['levels']]
    coords, kp = graph_gen.multi_layer_downsampling_select(g['xyz'], float(g['base_voxel_size']), levels)
    cents = graph_gen.multi_layer_downsampling(g['xyz'], float(g['base_voxel_size']), levels)
    assert coords[0].dtype == np.float32 and kp[0].dtype == np.int64 and kp[0].shape[1] == 1
    for i in range(len(levels)):
        assert np.array_equal(kp[i][:, 0], g['kp_%d' % i]), i
        assert np.array_equal(coords[i + 1], g['coords_%d' % (i + 1)]), i
        assert cents[i + 1].dtype == np.float64 or i == 2
        assert np.array_equal(np.asarray(cents[i + 1], dtype=np.float64), g['centroids_%d' % (i + 1)]), i


def test_multiscale_graph_batched_vs_oracle():
    """A three-level graph with two distinct scales, several frames in one call (frame_ptr), against the oracle frame
    by frame with the batch_data offsets (train.py:135-171)."""
    from pointgnn_b200.models import graph_gen
    cfg = [
        {'graph_gen_kwargs': {'num_neighbors': -1, 'radius': 1.0}, 'graph_gen_method': 'disjointed_rnn_local_graph_v3',
         'graph_level': 0, 'graph_scale': 1},
        {'graph_gen_kwargs': {'num_neighbors': -1, 'radius': 2.5}, 'graph_gen_method': 'disjointed_rnn_local_graph_v3',
         'graph_level': 1, 'graph_scale': 2.5},
        {'graph_gen_kwargs': {'num_neighbors': -1, 'radius': 4.0}, 'graph_gen_method': 'disjointed_rnn_local_graph_v3',
         'graph_level': 2, 'graph_scale': 2.5},
    ]
    clouds = [synth.lidar_frame(40 + i, n)[0] for i, n in enumerate((3000, 1, 2500))]
    fp = np.concatenate([[0], np.cumsum([len(c) for c in clouds])]).astype(np.int32)
    coords, kp, edges, fps = graph_gen.gen_multi_level_local_graph_v3(
        np.vstack(clouds), 0.5, cfg, frame_ptr=fp, return_frame_ptr=True)
    off = [0, 0, 0, 0]
    eo = [0, 0, 0]
    for c in clouds:
        co, ko, ed = graph.gen_multi_level_local_graph_v3(c, 0.5, cfg)
        for lvl in range(3):
            n_prev, n_cur = len(co[lvl]), len(co[lvl + 1])
            assert np.array_equal(coords[lvl + 1][off[lvl + 1]:off[lvl + 1] + n_cur], co[lvl + 1])
            assert np.array_equal(kp[lvl][off[lvl + 1]:off[lvl + 1] + n_cur, 0], ko[lvl][:, 0] + off[lvl])
            e = ed[lvl] + np.array([[off[lvl], off[lvl + 1]]])
            assert np.array_equal(edges[lvl][eo[lvl]:eo[lvl] + len(e)], e), lvl
            eo[lvl] += len(e)
        for lvl in range(4):
            off[lvl] += len(co[lvl])
    for lvl in range(3):
        assert eo[lvl] == len(edges[lvl])
        assert int(fps[lvl + 1][-1]) == len(coords[lvl + 1])


def test_scaled_radius_graph_vs_reference_golden():
    """gen_disjointed_rnn_local_graph_v3(..., scale=[sx, sy, sz]) (graph_gen.py:203-206: float64 division of both point
    sets before the ball tree) - bit-exact against the reference's own output, directly and through a level config."""
    import os
    from pointgnn_b200.models import graph_gen
    g = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'graph_scale.npz'))
    for i in range(3):
        scale = [float(v) for v in g['scale_%d' % i]]
        e = graph_gen.gen_disjointed_rnn_local_graph_v3(g['xyz'], g['centers'], float(g['radius']), -1, scale=scale)
        assert e.dtype == np.int64 and np.array_equal(e, g['edges_%d' % i]), i
    # unscaled call unchanged, scale of ones identical to it
    e1 = graph_gen.gen_disjointed_rnn_local_graph_v3(g['xyz'], g['centers'], 1.0, -1)
    e2 = graph_gen.gen_disjointed_rnn_local_graph_v3(g['xyz'], g['centers'], 1.0, -1, scale=[1.0, 1.0, 1.0])
    assert np.array_equal(e1, e2) and np.array_equal(e1, graph.gen_disjointed_rnn_local_graph_v3(g['xyz'], g['centers'], 1.0, -1))
    cfg = [{'graph_gen_kwargs': {'num_neighbors': -1, 'radius': 1.0, 'scale': [1.0, 0.5, 1.0]},
            'graph_gen_method': 'disjointed_rnn_local_graph_v3', 'graph_level': 0, 'graph_scale': 1},
           {'graph_gen_kwargs': {'num_neighbors': -1, 'radius': 4.0, 'scale': [1.0, 0.5, 1.0]},
            'graph_gen_method': 'disjointed_rnn_local_graph_v3', 'graph_level': 1, 'graph_scale': 1}]
    xyz, _ = synth.lidar_frame(33, 5000)
    got = graph_gen.gen_multi_level_local_graph_v3(xyz, 0.8, cfg)
    want = graph.gen_multi_level_local_graph_v3(xyz, 0.8, cfg)
    for a, b in zip(got[2], want[2]):
        assert np.array_equal(a, b)
    with pytest.raises(ValueError):
        graph_gen.gen_disjointed_rnn_local_graph_v3(g['xyz'], g['centers'], 1.0, -1, scale=[1.0, 0.0, 1.0])


def test_rnd3d_centroid_downsampling_vs_reference_golden():
    """add_rnd3d=True with the centroid method (graph_gen.py:24-39, 82-88) against the reference's own output for the same
    seeded np.random draws.  The reference sums a voxel's points in float32 in argsort order, the kernel in fp64: voxel
    membership, order and count must be equal, centroids within 1e-4 m, and every snapped vertex must be a nearest
    vertex of its centroid within that tolerance (two-point voxels are exact ties upstream)."""
    import os
    from pointgnn_b200.models import graph_gen
    g = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'graph_rnd3d.npz'))
    levels = [float(v) for v in g['levels']]
    xyz, voxel = g['xyz'], float(g['base_voxel_size'])
    np.random.seed(int(g['seed']))
    cents = graph_gen.multi_layer_downsampling(xyz, voxel, levels, add_rnd3d=True)
    for i in range(len(levels)):
        want = g['centroids_%d' % (i + 1)]
        assert cents[i + 1].shape == want.shape, i
        assert np.abs(np.asarray(cents[i + 1], dtype=np.float64) - want).max() < 1e-4, i
    np.random.seed(int(g['seed']))
    coords, kp = graph_gen.multi_layer_downsampling_select(xyz, voxel, levels, add_rnd3d=True)
    assert np.array_equal(kp[1][:, 0], np.arange(len(kp[0])))                       # same scale: identity
    for i in (0, 2):
        base = np.asarray(coords[i], dtype=np.float64)
        cent = g['centroids_%d' % (i + 1)]
        assert len(kp[i]) == len(cent)
        assert np.array_equal(coords[i + 1], coords[i][kp[i][:, 0]])
        d_mine = np.linalg.norm(base[kp[i][:, 0]] - cent, axis=1)
        d_best = np.empty(len(cent))
        for s0 in range(0, len(cent), 256):
            d_best[s0:s0 + 256] = np.sqrt(((cent[s0:s0 + 256, None, :] - base[None, :, :]) ** 2).sum(2)).min(1)
        assert np.all(d_mine <= d_best + 2e-4), i
    # index agreement is high but not total: every two-point voxel is an exact tie upstream (about one voxel in ten),
    # broken by float32 rounding noise in the reference and by the exact fp64 distance here
    assert (kp[0][:, 0] == g['kp_0']).mean() > 0.85
    # through the graph generator (what train.py would call with downsample_method='center', add_rnd3d=True)
    cfg = [{'graph_gen_kwargs': {'num_neighbors': -1, 'radius': 1.0}, 'graph_gen_method': 'disjointed_rnn_local_graph_v3',
            'graph_level': 0, 'graph_scale': 1},
           {'graph_gen_kwargs': {'num_neighbors': -1, 'radius': 4.0}, 'graph_gen_method': 'disjointed_rnn_local_graph_v3',
            'graph_level': 1, 'graph_scale': 1}]
    np.random.seed(3)
    co, kpi, ed = graph_gen.gen_multi_level_local_graph_v3(xyz, 0.8, cfg, add_rnd3d=True)
    want_e = graph.gen_disjointed_rnn_local_graph_v3(co[0], co[1], 1.0, -1)
    assert np.array_equal(ed[0], want_e) and np.array_equal(co[1], xyz[kpi[0][:, 0]])


def test_random_keypoints_vs_reference_golden():
    """The training-time keypoints (graph_gen.py:92-153) fed the random numbers recorded in tests/golden/graph_random.npz
    (the reference's own function with its generators patched to them): same voxels, first-appearance order, same
    member, with the float32 voxel rule and with the shifted float64 one (add_rnd3d)."""
    import os
    from pointgnn_b200.models import graph_gen
    g = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'graph_random.npz'))
    cloud = graph_gen._Cloud(torch.from_numpy(g['xyz']).cuda())
    for tag, add in (('plain', False), ('rnd3d', True)):
        u = torch.from_numpy(g['u_' + tag]).cuda()
        coords, kp, fps = graph_gen._downsampling_random(cloud, 0.8, [1, 1], add, uniform=[u, None],
                                                         shifts=[g['shift_' + tag], None])
        want = g['kp_' + tag]
        assert np.array_equal(_np(kp[0][:, 0]), want), tag
        assert np.array_equal(_np(coords[1]), g['xyz'][want]), tag
        assert _np(fps[1]).tolist() == [0, len(want)], tag
        assert np.array_equal(_np(kp[1][:, 0]), np.arange(len(want))), tag


def test_neighbor_cap_invariants_and_seed(car):
    """The random neighbour cap (graph_gen.py:210-214) on a real level-0 radius graph: rows of at most num_neighbors
    entries unchanged, longer rows exactly num_neighbors distinct true neighbours; the same seed gives the same edges."""
    from pointgnn_b200.models import graph_gen
    xyz, _ = synth.lidar_frame(17, 8000)
    t = torch.from_numpy(xyz).cuda()
    coords, _, _, fps = graph_gen.gen_multi_level_local_graph_v3(t, return_frame_ptr=True, **car.graph_kwargs)
    r0 = car.graph_kwargs['level_configs'][0]['graph_gen_kwargs']['radius']
    full = graph_gen._radius_edges(t, fps[0], coords[1], fps[1], r0, -1)
    capped = graph_gen._radius_edges(t, fps[0], coords[1], fps[1], r0, 8, cap_seed=1234)
    again = graph_gen._radius_edges(t, fps[0], coords[1], fps[1], r0, 8, cap_seed=1234)
    full_np, capped_np = _np(full).astype(np.int64), _np(capped).astype(np.int64)
    assert np.array_equal(full_np, graph.radius_graph(xyz, _np(coords[1]), r0))
    assert graph.check_neighbor_cap(full_np, capped_np, 8) > 0
    assert np.array_equal(_np(again), _np(capped))


def test_radius_graph_capacity_contract_by_name():
    """pg_radius_graph with an edge buffer that is too small: PG_ERR_CAPACITY, the exact E, and a valid row_ptr."""
    import ctypes
    from pointgnn_b200 import _lib
    xyz, _ = synth.lidar_frame(12, 4000)
    pts = torch.from_numpy(xyz).cuda()
    ctr = pts[::5].contiguous()
    fp = torch.tensor([0, pts.shape[0]], dtype=torch.int32, device='cuda')
    cfp = torch.tensor([0, ctr.shape[0]], dtype=torch.int32, device='cuda')
    row_ptr, edges = _lib.radius_graph(pts, fp, ctr, cfp, 1.0)
    assert np.array_equal(_np(edges.t()).astype(np.int64), graph.radius_graph(xyz, xyz[::5], 1.0))
    rp = torch.full_like(row_ptr, -1)
    buf = torch.empty((2, 1), dtype=torch.int32, device='cuda')
    e = ctypes.c_int64(0)
    with pytest.raises(_lib.PointGNNError) as err:
        _lib._call('pg_radius_graph', points=pts, point_frame_ptr=fp, centers=ctr, center_frame_ptr=cfp, num_frames=1,
                   num_points=pts.shape[0], num_centers=ctr.shape[0], radius=1.0, out_row_ptr=rp, out_src=buf[0],
                   out_dst=buf[1], capacity=1, out_num_edges_host=ctypes.byref(e))
    assert err.value.code == _lib.PG_ERR_CAPACITY
    assert e.value == edges.shape[1] > 1
    assert torch.equal(rp, row_ptr)


def test_multi_level_graph_capacity_retry(car):
    """_lib.multi_level_graph started with a keypoint buffer below K, then with edge buffers below E0 / E1: the retry
    loop must end with the result of a fresh call, which equals the oracle."""
    from pointgnn_b200 import _lib
    from pointgnn_b200.models import graph_gen
    xyz, _ = synth.lidar_frame(13, 6000)
    t = torch.from_numpy(xyz).cuda()
    fp = torch.tensor([0, xyz.shape[0]], dtype=torch.int32, device='cuda')
    kw = car.graph_kwargs
    voxel = graph_gen._voxel_vector(kw['base_voxel_size'], kw['level_configs'][0]['graph_scale'])
    r0, r1 = (c['graph_gen_kwargs']['radius'] for c in kw['level_configs'])
    key = (t.device.index, int(xyz.shape[0]), tuple(float(v) for v in voxel), float(r0), float(r1))
    _lib._graph_capacity.pop(key, None)
    fresh = _lib.multi_level_graph(t, fp, voxel, r0, r1)
    k, e0, e1 = fresh[0].numel(), fresh[3].shape[1], fresh[4].shape[1]
    _, kp_o, edges_o = graph.gen_multi_level_local_graph_v3(xyz, **kw)
    assert np.array_equal(_np(fresh[0]), kp_o[0][:, 0])
    assert np.array_equal(_np(fresh[3].t()).astype(np.int64), edges_o[0])
    assert np.array_equal(_np(fresh[4].t()).astype(np.int64), edges_o[1])
    n = xyz.shape[0]
    try:
        for caps in ((k // 2, 32 * n, 48 * n), (k, e0 // 2, e1), (k, e0, e1 // 2)):
            _lib._graph_capacity[key] = caps
            got = _lib.multi_level_graph(t, fp, voxel, r0, r1)
            for a, b in zip(got, fresh):
                assert torch.equal(a, b), caps
    finally:
        _lib._graph_capacity.pop(key, None)
