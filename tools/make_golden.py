"""Generate tests/golden/* (run in the BUILD container, where /root/reference exists).

* weights_<cfg>.npz / config_<cfg>.json : the reference's trained checkpoints
  (checkpoints/<cfg>/model-*.{index,data}) decoded with utils/tf_checkpoint.py, and the frozen
  JSON config saved beside them (train.py:591-592).  Data, not code.
* graph_<cfg>.npz : a seeded synthetic frame, the keypoints of the oracle's voxel restatement,
  and the edge lists produced by the REFERENCE's own models/graph_gen.py
  (gen_disjointed_rnn_local_graph_v3, scikit-learn ball tree) on those vertices, in canonical
  (dst, src) order -> pins oracle/graph.py and the CUDA radius kernels to the reference.
* gnn_<cfg>.npz : logits / box encodings / class probabilities / per-layer features obtained by
  executing the REFERENCE'S OWN saved TensorFlow graph (checkpoints/<cfg>/model-N.meta, the
  MetaGraphDef train.py wrote) with the NumPy GraphDef interpreter oracle/graphdef.py on that
  frame with the real weights -> pins oracle/gnn.py and the CUDA kernels to the graph the
  reference built (op order, concat order, gather indices, segment ids), for all seven shipped
  checkpoints.  The script asserts that oracle/gnn.py reproduces those vectors to <= 1e-5.
* graph_live_reference.npz : the reference's radius graphs on a second seeded frame (two voxel / radius settings).
* checkpoints/<cfg>/ : index and state file of each shipped checkpoint (+ two gzipped saved graphs), from which
  oracle/checkpoint_fixture.py rebuilds the checkpoints with the weights above.
"""
import glob
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import gnn, graph, graphdef, reference_graph, synth  # noqa: E402
from pointgnn_b200.utils import tf_checkpoint  # noqa: E402

GOLDEN = os.path.join(ROOT, 'tests', 'golden')
CONFIGS = {
    'car_auto_T3_train': dict(num_points=3000, frame=7, graph='car_auto_T3_train'),
    'ped_cyl_auto_T3_trainval': dict(num_points=3000, frame=8, graph='ped_cyl_auto_T3_trainval'),
    # the other shipped checkpoints share car_auto_T3_train's graph settings (and its graph fixture)
    'car_auto_T0_train': dict(num_points=3000, frame=7, graph='car_auto_T3_train'),
    'car_auto_T1_train': dict(num_points=3000, frame=7, graph='car_auto_T3_train'),
    'car_auto_T2_train': dict(num_points=3000, frame=7, graph='car_auto_T3_train'),
    'car_auto_T3_trainval': dict(num_points=3000, frame=7, graph='car_auto_T3_train'),
    'car_fixed_T3_train': dict(num_points=3000, frame=7, graph='car_auto_T3_train'),
}


def main():
    os.makedirs(GOLDEN, exist_ok=True)
    ref = reference_graph.load()
    for name, spec in CONFIGS.items():
        ckpt_dir = os.path.join(reference_graph.REFERENCE_ROOT, 'checkpoints', name)
        with open(os.path.join(ckpt_dir, 'config')) as f:
            config = json.load(f)
        with open(os.path.join(GOLDEN, 'config_%s.json' % name), 'w') as f:
            json.dump(config, f, indent=1, sort_keys=True)
        weights = {k: v for k, v in tf_checkpoint.load_checkpoint(ckpt_dir).items()
                   if k.endswith('/weights') or k.endswith('/biases')}
        np.savez(os.path.join(GOLDEN, 'weights_%s.npz' % name), **weights)

        xyz, intensity = synth.lidar_frame(spec['frame'], spec['num_points'])
        kw = config['runtime_graph_gen_kwargs']
        coords, keypoints, edges = graph.gen_multi_level_local_graph_v3(xyz, **kw)
        ref_edges = []
        for lvl, cfg in enumerate(kw['level_configs']):
            e = ref.gen_disjointed_rnn_local_graph_v3(coords[lvl], coords[lvl + 1], **cfg['graph_gen_kwargs'])
            assert np.all(np.diff(e[:, 1]) >= 0), 'reference edges are not grouped by destination'
            e = graph.canonical_edges(e)
            assert np.array_equal(e, edges[lvl]), 'oracle radius graph != reference graph_gen'
            ref_edges.append(e.astype(np.int32))
        if spec['graph'] == name:
            np.savez_compressed(
                os.path.join(GOLDEN, 'graph_%s.npz' % name), xyz=xyz, intensity=intensity,
                keypoint_idx=keypoints[0][:, 0].astype(np.int32),
                edges0=ref_edges[0], edges1=ref_edges[1])
        # the reference's own saved graph, interpreted op by op
        meta = sorted(glob.glob(os.path.join(ckpt_dir, 'model-*.meta')))[-1]
        nodes = graphdef.load_meta_graph(meta)
        pool_node = 'layer1/combined_features/fully_connected_1/Relu'
        last_node = nodes['output/predictor/cls/fully_connected/MatMul'].inputs[0]
        all_vars = tf_checkpoint.load_checkpoint(ckpt_dir)
        out = graphdef.run_forward(meta, all_vars, intensity, coords, keypoints, edges,
                                   extra_nodes=(pool_node, last_node))
        np.savez_compressed(os.path.join(GOLDEN, 'gnn_%s.npz' % name), logits=out['logits'], boxes=out['boxes'],
                            probs=out['probs'], features_pool=out[pool_node], features_last=out[last_node])
        with open(os.path.join(GOLDEN, 'graphdef_ops_%s.json' % name), 'w') as f:
            json.dump({'meta': os.path.basename(meta), 'nodes_total': len(nodes), 'ops_executed': out['ops']},
                      f, indent=1, sort_keys=True)
        logits, boxes, feats = gnn.predict(weights, config['model_kwargs']['layer_configs'],
                                           config['num_classes'], 7, intensity, coords, keypoints, edges,
                                           return_features=True)
        err = max(np.abs(logits - out['logits']).max(), np.abs(boxes - out['boxes']).max(),
                  np.abs(feats[1] - out[pool_node]).max(), np.abs(feats[-1] - out[last_node]).max())
        assert err <= 1e-5, 'oracle/gnn.py differs from the reference graph by %g' % err
        print(name, 'K=%d E0=%d E1=%d' % (len(keypoints[0]), len(edges[0]), len(edges[1])),
              'logits', logits.shape, float(np.abs(logits).max()), 'restatement-vs-graphdef %g' % err)


POST_CASES = [   # (name, label_method, num_classes, nms_overlapped_thres of the shipped config, seed)
    ('car', 'Car', 4, 0.01, 11),
    ('ped', 'Pedestrian_and_Cyclist', 6, 0.2, 12),
]


def post_goldens():
    """tests/golden/post_<case>.npz: run.py:265-325 executed with the reference's own box_encoding.py and nms.py
    (shapely replaced by the convex-polygon stand-in of oracle/postprocess.py) on seeded synthetic network outputs."""
    from oracle import postprocess as pp
    be, nms = pp.reference_modules()
    for name, method, c, thres, seed in POST_CASES:
        pts, enc, probs = pp.synthetic_outputs(seed, num_classes=c)
        out = {'points_xyz': pts, 'box_encodings': enc, 'probs': probs, 'thres': np.float64(thres)}
        for variant in ('uncertainty', 'merge_only', 'score_only', 'plain'):
            r = pp.reference_postprocess_frame(be, nms, probs.copy(), enc.copy(), pts.copy(), method, thres, variant)
            for k in ('label', 'box', 'score', 'nms_index'):
                out['%s_%s' % (variant, k)] = r[k]
            out['cand_index'] = r['cand_index']
            out['decoded'] = r['decoded']
        np.savez_compressed(os.path.join(GOLDEN, 'post_%s.npz' % name), **out)
        print('post', name, 'candidates', len(out['cand_index']), 'kept', len(out['uncertainty_label']))


BOX_CANONICAL_ROWS = 600


def box_canonical_inputs(label_method, seed, rows=BOX_CANONICAL_ROWS):
    """Seeded inputs of the canonical box decoder for one label map: every label of the map (Background and DontCare
    included) on rows [M, 1] int32, vertices [M, 3] float32 (a quarter of them hundreds of metres out) and
    encodings [M, 2, 7] float32 with |e6| up to 4 (slot 1 is only offset by the vertex)."""
    from oracle import postprocess as pp
    num_labels = max(pp.LABEL_MAPS[label_method].values()) + 1
    rng = np.random.default_rng(seed)
    labels = (np.arange(rows) % num_labels).astype(np.int32)[:, None]
    xyz = np.c_[rng.uniform(-40, 40, rows), rng.uniform(-3, 3, rows), rng.uniform(0, 70, rows)]
    xyz[: rows // 4] *= rng.uniform(5, 20, (rows // 4, 1))
    enc = rng.standard_normal((rows, 2, 7))
    enc[:, :, 3:6] *= 0.5
    enc[:, :, 6] = rng.uniform(-4, 4, (rows, 2))
    return labels, xyz.astype(np.float32), enc.astype(np.float32)


def box_canonical_goldens():
    """tests/golden/box_canonical.npz: the reference's own classaware_all_class_box_canonical_decoding
    (box_encoding.py:345-395) on box_canonical_inputs for the three label maps of run.py."""
    from oracle import postprocess as pp
    be, _ = pp.reference_modules()
    out = {}
    for seed, method in enumerate(sorted(pp.LABEL_MAPS)):
        labels, xyz, enc = box_canonical_inputs(method, 100 + seed)
        dec = be.classaware_all_class_box_canonical_decoding(labels, xyz, enc, pp.LABEL_MAPS[method])
        assert dec.dtype == np.float32
        out.update({'labels_' + method: labels, 'xyz_' + method: xyz, 'enc_' + method: enc, 'dec_' + method: dec})
        print('box_canonical', method, 'rows', len(labels))
    np.savez_compressed(os.path.join(GOLDEN, 'box_canonical.npz'), **out)


def kitti_goldens():
    """tests/golden/kitti_io.npz + kitti_result_car.txt: the reference's own dataset/kitti_dataset.py (Open3D stubbed)
    on a synthetic KITTI-format frame - calibration matrices, camera points in image with colours - and run.py:361-429
    (label conversion + file text) assembled from the reference's functions on the post_car detections."""
    import tempfile
    import cv2
    from oracle import kitti as ok
    from oracle import postprocess as pp
    ref = ok.reference_dataset_module()
    be, nms = pp.reference_modules()
    root = tempfile.mkdtemp()
    ok.write_synthetic_kitti(root, [5], 6000)
    ds = ref.KittiDataset(os.path.join(root, 'image/testing/image_2'), os.path.join(root, 'velodyne/testing/velodyne/'),
                          os.path.join(root, 'calib/testing/calib/'), '', num_classes=4, is_training=False)
    calib = ds.get_calib(0)
    pts = ds.get_cam_points_in_image_with_rgb(0, None)
    velo = np.fromfile(os.path.join(root, 'velodyne/testing/velodyne/000000.bin'), dtype=np.float32).reshape(-1, 4)
    image = cv2.imread(os.path.join(root, 'image/testing/image_2/000000.png'))
    # run.py:361-429 with the reference's functions, on the car post-processing fixture
    g = dict(np.load(os.path.join(GOLDEN, 'post_car.npz')))
    labels, boxes, scores = g['uncertainty_label'], g['uncertainty_box'], g['uncertainty_score']
    cand_xyz = g['points_xyz'][g['cand_index'] // 4]

    def occlusion(label, xyz):            # run.py:88-100
        if xyz.shape[0] == 0:
            return 0
        normals, lower, upper = ds.box3d_to_normals(label)
        projected = np.matmul(xyz, np.transpose(normals))
        rates = [(np.max(projected[:, i]) - np.min(projected[:, i])) / (upper[i] - lower[i]) for i in range(3)]
        return rates[0] * rates[1] * rates[2]

    corners_all = nms.boxes_3d_to_corners(boxes)
    names = ['Background', 'Car', 'Car', 'DontCare']
    text = ''
    for i in range(len(corners_all)):
        corners_xy = ds.cam_points_to_image(ref.Points(xyz=corners_all[i], attr=None), calib).xyz[:, :2]
        xmin, ymin = np.amin(corners_xy, axis=0)
        xmax, ymax = np.amax(corners_xy, axis=0)
        clip_xmin, clip_ymin, clip_xmax, clip_ymax = max(xmin, 0.0), max(ymin, 0.0), min(xmax, 1242.0), min(ymax, 375.0)
        truncation_rate = 1.0 - (clip_ymax - clip_ymin) * (clip_xmax - clip_xmin) / ((ymax - ymin) * (xmax - xmin))
        if truncation_rate > 0.4:
            continue
        x3d, y3d, z3d, l, h, w, yaw = boxes[i]
        tmp_label = {"x3d": x3d, "y3d": y3d, "z3d": z3d, "yaw": yaw, "height": h, "width": w, "length": l}
        inside_mask = ds.sel_xyz_in_box3d(tmp_label, cand_xyz)
        score = (1 + occlusion(tmp_label, cand_xyz[inside_mask])) * scores[i]
        for field in (names[labels[i]], -1, -1, 0, clip_xmin, clip_ymin, clip_xmax, clip_ymax, h, w, l, x3d, y3d, z3d, yaw, score):
            text += str(field) + ' '
        text += '\n'
    text += '\n'
    with open(os.path.join(GOLDEN, 'kitti_result_car.txt'), 'w') as f:
        f.write(text)
    np.savez_compressed(os.path.join(GOLDEN, 'kitti_io.npz'), velo=velo, image=image, xyz=pts.xyz, attr=pts.attr,
                        **{'calib_' + k: np.asarray(calib[k]) for k in ('velo_to_cam', 'cam_to_image', 'cam_to_velo', 'P2')})
    with open(os.path.join(GOLDEN, 'kitti_calib.txt'), 'w') as f:
        f.write(ok.CALIB_TEXT)
    print('kitti: points in image', pts.xyz.shape, 'result lines', text.count('\n') - 1)


VOXEL_AVG_SIZES = (0.1, 0.4)


def kitti_voxel_avg_goldens():
    """tests/golden/kitti_voxel_avg.npz: the reference's own get_cam_points / get_cam_points_in_image_with_rgb
    (kitti_dataset.py:611-627, 666-689, with downsample_by_average_voxel :16-48) on the synthetic frame of kitti_io.npz,
    for two voxel sizes.  Per size <s>: keys_<s> / counts_<s> (the occupied voxels, recomputed from the reference's own
    index arithmetic), mean_xyz_<s> / mean_attr_<s> (its float64 means), crop_index_<s> (ranks of the voxels that
    survive its crop), crop_xyz_<s> / crop_attr_<s> (its result), and crop_unsure_<s> / pixel_unsure_<s>: ranks whose
    crop verdict / colour pixel changes when the mean moves by 1e-4 (oracle.voxel_average.decision_margin)."""
    import cv2
    from oracle import kitti as ok
    from oracle import voxel_average as ova
    ref = ok.reference_dataset_module()
    root = tempfile.mkdtemp()
    ok.write_synthetic_kitti(root, [5], 6000)
    ds = ref.KittiDataset(os.path.join(root, 'image/testing/image_2'), os.path.join(root, 'velodyne/testing/velodyne/'),
                          os.path.join(root, 'calib/testing/calib/'), '', num_classes=4, is_training=False)
    io = np.load(os.path.join(GOLDEN, 'kitti_io.npz'))
    velo = np.fromfile(os.path.join(root, 'velodyne/testing/velodyne/000000.bin'), dtype=np.float32).reshape(-1, 4)
    image = cv2.imread(os.path.join(root, 'image/testing/image_2/000000.png'))
    assert np.array_equal(velo, io['velo']) and np.array_equal(image, io['image']), 'not the frame of kitti_io.npz'
    calib = ds.get_calib(0)
    height, width = image.shape[:2]
    out = {}
    for vs in VOXEL_AVG_SIZES:
        tag = ('%g' % vs).replace('.', 'p')
        full = ds.get_cam_points(0)
        avg = ds.get_cam_points(0, downsample_voxel_size=vs)
        crop = ds.get_cam_points_in_image_with_rgb(0, vs)
        keys, _ = ova.voxel_keys(full.xyz, vs)
        unique_keys, counts = np.unique(keys, return_counts=True)
        assert len(unique_keys) == len(avg.xyz) and avg.xyz.dtype == np.float64
        keep, _ = ova.crop_mask(avg.xyz, calib, width, height)
        assert np.array_equal(avg.xyz[keep], crop.xyz), 'restated crop != reference crop'
        crop_unsure, pixel_unsure = ova.decision_margin(avg.xyz, calib, width, height)
        out.update({'keys_' + tag: unique_keys, 'counts_' + tag: counts, 'mean_xyz_' + tag: avg.xyz,
                    'mean_attr_' + tag: avg.attr, 'crop_index_' + tag: np.flatnonzero(keep), 'crop_xyz_' + tag: crop.xyz,
                    'crop_attr_' + tag: crop.attr, 'crop_unsure_' + tag: np.flatnonzero(crop_unsure),
                    'pixel_unsure_' + tag: np.flatnonzero(pixel_unsure)})
        print('kitti_voxel_avg', vs, 'points', len(full.xyz), 'voxels', len(unique_keys), 'in image', len(crop.xyz),
              'crop unsure', int(crop_unsure.sum()), 'pixel unsure', int(pixel_unsure.sum()))
    np.savez_compressed(os.path.join(GOLDEN, 'kitti_voxel_avg.npz'), **out)


def graph_random_goldens():
    """tests/golden/graph_random.npz: the reference's OWN multi_layer_downsampling_random (graph_gen.py:92-153) with its
    two random sources patched to recorded numbers: np.random.random -> `shift`, random.choice(seq) ->
    seq[floor(u[o] * len(seq))] for the o-th call.  The CUDA path gets the same numbers as arguments and must return
    the same keypoints, with and without add_rnd3d."""
    import random as _random
    ref = reference_graph.load()
    xyz, _ = synth.lidar_frame(3, 8000)
    rng = np.random.default_rng(0)
    out = {'xyz': xyz}
    for add in (False, True):
        shift = rng.random((1, 3))
        u = rng.random(len(xyz)).astype(np.float32)
        counter = {'o': 0}

        def fake_choice(seq):
            o = counter['o']
            counter['o'] += 1
            return seq[min(int(np.float32(u[o]) * np.float32(len(seq))), len(seq) - 1)]

        orig_choice, orig_rand = _random.choice, np.random.random
        _random.choice = fake_choice
        np.random.random = lambda size=None: shift.copy()
        try:
            vc, kp = ref.multi_layer_downsampling_random(xyz, 0.8, [1, 1], add_rnd3d=add)
        finally:
            _random.choice, np.random.random = orig_choice, orig_rand
        tag = 'rnd3d' if add else 'plain'
        out['shift_' + tag] = shift
        out['u_' + tag] = u
        out['kp_' + tag] = kp[0][:, 0].astype(np.int32)
        vc2, kp2 = graph.multi_layer_downsampling_random(xyz, 0.8, [1, 1], add_rnd3d=add, shifts=[shift, None],
                                                         uniforms=[u, None])
        assert np.array_equal(kp[0], kp2[0]) and np.array_equal(vc[1], vc2[1]), 'oracle restatement != reference'
        print('graph_random', tag, 'keypoints', len(kp[0]))
    np.savez_compressed(os.path.join(GOLDEN, 'graph_random.npz'), **out)


def graph_multiscale_goldens():
    """tests/golden/graph_multiscale.npz: the reference's OWN multi_layer_downsampling_select (graph_gen.py:49-90, with
    multi_layer_downsampling :11-47) for SEVERAL distinct scales - which cloud is voxelised, which level is searched,
    the index layout are the reference running.  Two calls inside it have an UNSPECIFIED order upstream and are
    canonicalised: (1) open3d.voxel_down_sample (:41-45; Open3D 0.7 is not installable) is served by the oracle's
    restated voxel rule (ascending voxel key); (2) the kd_tree 1-NN (:84-86) is scikit-learn's own query, but where
    several base vertices are EXACTLY equidistant in fp64 - every voxel with two points: its centroid is their
    midpoint - scikit-learn returns whichever its tree visits first (version dependent); the wrapper returns the
    lowest index among those exact minimisers.  The fixture records how many rows needed (2)."""
    import sys as _sys
    from sklearn.neighbors import NearestNeighbors as _SkNN
    ref = reference_graph.load()
    o3d = _sys.modules['open3d']

    class _Pcd(object):
        points = None
    o3d.PointCloud = _Pcd
    o3d.Vector3dVector = lambda a: np.asarray(a)
    o3d.voxel_down_sample = lambda pcd, voxel_size: type('R', (), {'points': graph.voxel_down_sample(pcd.points, voxel_size)})()
    stats = {'queries': 0, 'ties': 0}

    class _CanonicalTies(object):
        def __init__(self, n_neighbors=1, algorithm='kd_tree', n_jobs=1):
            assert n_neighbors == 1 and algorithm == 'kd_tree'
            self._nn = _SkNN(n_neighbors=1, algorithm=algorithm, n_jobs=n_jobs)

        def fit(self, x):
            self._x = np.asarray(x, dtype=np.float64)
            self._nn.fit(x)
            return self

        def kneighbors(self, q, return_distance=False):
            assert not return_distance
            dist, idx = self._nn.kneighbors(q, return_distance=True)
            q64 = np.asarray(q, dtype=np.float64)
            out = idx.copy()
            for j in range(len(q64)):
                c = self._nn.radius_neighbors(q64[j:j + 1], radius=dist[j, 0] * (1 + 1e-9) + 1e-12,
                                              return_distance=False)[0]
                d = self._x[c] - q64[j]
                d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
                best = np.sort(c[d2 == d2.min()])
                assert idx[j, 0] in best, 'scikit-learn returned a non-minimiser'
                stats['queries'] += 1
                stats['ties'] += int(len(best) > 1)
                out[j, 0] = best[0]
            return out

    xyz, _ = synth.lidar_frame(11, 12000)
    levels = [1, 2, 2, 4.5]
    orig = ref.NearestNeighbors
    ref.NearestNeighbors = _CanonicalTies
    try:
        vc, kp = ref.multi_layer_downsampling_select(xyz, 0.4, levels)
    finally:
        ref.NearestNeighbors = orig
    vo, ko = graph.multi_layer_downsampling_select(xyz, 0.4, levels)
    out = {'xyz': xyz, 'levels': np.asarray(levels, dtype=np.float64), 'base_voxel_size': np.float64(0.4),
           'tie_rows': np.int64(stats['ties']), 'query_rows': np.int64(stats['queries'])}
    for i in range(len(levels)):
        assert np.array_equal(np.asarray(vc[i + 1]), np.asarray(vo[i + 1])), 'oracle coordinates != reference (level %d)' % i
        assert np.array_equal(np.asarray(kp[i]), np.asarray(ko[i])), 'oracle index != reference (level %d)' % i
        out['coords_%d' % (i + 1)] = np.asarray(vc[i + 1], dtype=np.float32)
        out['kp_%d' % i] = np.asarray(kp[i])[:, 0].astype(np.int32)
        print('graph_multiscale level', i, 'scale', levels[i], 'vertices', len(kp[i]))
    print('graph_multiscale: %d of %d 1-NN queries had exactly tied minimisers' % (stats['ties'], stats['queries']))
    cents = ref.multi_layer_downsampling(xyz, 0.4, levels)
    for i in range(len(levels)):
        out['centroids_%d' % (i + 1)] = np.asarray(cents[i + 1], dtype=np.float64)
    np.savez_compressed(os.path.join(GOLDEN, 'graph_multiscale.npz'), **out)


def graph_scale_goldens():
    """tests/golden/graph_scale.npz: the reference's OWN gen_disjointed_rnn_local_graph_v3 with the per-axis `scale`
    argument (graph_gen.py:203-206; float64 division before the ball tree), rows in canonical order."""
    ref = reference_graph.load()
    xyz, _ = synth.lidar_frame(21, 3000)
    centers = xyz[::7].copy()
    out = {'xyz': xyz, 'centers': centers, 'radius': np.float64(1.0)}
    for i, scale in enumerate(([1.0, 0.7, 1.3], [0.3, 1.0, 1.9], [2.0, 2.0, 2.0])):
        e = ref.gen_disjointed_rnn_local_graph_v3(xyz, centers, 1.0, -1, scale=scale)
        e = e[np.lexsort((e[:, 0], e[:, 1]))]
        assert np.array_equal(e, graph.gen_disjointed_rnn_local_graph_v3(xyz, centers, 1.0, -1, scale=scale)), 'oracle != reference'
        out['scale_%d' % i] = np.asarray(scale, dtype=np.float64)
        out['edges_%d' % i] = e.astype(np.int32)
        print('graph_scale', scale, 'edges', len(e))
    np.savez_compressed(os.path.join(GOLDEN, 'graph_scale.npz'), **out)


def graph_rnd3d_goldens():
    """tests/golden/graph_rnd3d.npz: the reference's OWN multi_layer_downsampling / multi_layer_downsampling_select with
    add_rnd3d=True and the centroid method (graph_gen.py:24-39, 82-88), NumPy's global generator seeded; the oracle,
    seeded the same way, must return the same arrays bit for bit (it makes the same NumPy calls)."""
    ref = reference_graph.load()
    xyz, _ = synth.lidar_frame(17, 9000)
    levels = [1, 1, 2.5]
    np.random.seed(7)
    cents = ref.multi_layer_downsampling(xyz, 0.4, levels, add_rnd3d=True)
    np.random.seed(7)
    co = graph.multi_layer_downsampling(xyz, 0.4, levels, add_rnd3d=True)
    np.random.seed(7)
    vc, kp = ref.multi_layer_downsampling_select(xyz, 0.4, levels, add_rnd3d=True)
    np.random.seed(7)
    vo, ko = graph.multi_layer_downsampling_select(xyz, 0.4, levels, add_rnd3d=True)
    out = {'xyz': xyz, 'levels': np.asarray(levels, dtype=np.float64), 'base_voxel_size': np.float64(0.4), 'seed': np.int64(7)}
    exact = 0
    for i in range(len(levels)):
        assert np.array_equal(np.asarray(cents[i + 1]), np.asarray(co[i + 1])), 'oracle centroids != reference'
        # the kd-tree tie rule (lowest index among exact minimisers) only matters for exact ties; with float32-summed
        # centroids there are hardly any, but identical base rows (level 3) still tie
        same = np.asarray(kp[i])[:, 0] == np.asarray(ko[i])[:, 0]
        exact += int(same.sum())
        out['centroids_%d' % (i + 1)] = np.asarray(cents[i + 1], dtype=np.float64)
        out['kp_%d' % i] = np.asarray(kp[i])[:, 0].astype(np.int32)
        out['coords_%d' % (i + 1)] = np.asarray(vc[i + 1], dtype=np.float32)
        print('graph_rnd3d level', i, 'vertices', len(kp[i]), 'oracle index == reference:', int(same.sum()))
    np.savez_compressed(os.path.join(GOLDEN, 'graph_rnd3d.npz'), **out)


def graph_live_reference_goldens():
    """graph_live_reference.npz: the REFERENCE's gen_disjointed_rnn_local_graph_v3 (canonical edge order) on a seeded
    2 500-point frame, for the oracle's keypoints at two voxel / radius settings (both graph levels each)."""
    ref = reference_graph.load()
    xyz, _ = synth.lidar_frame(11, 2500)
    out = {}
    for i, (voxel, r0, r1) in enumerate(((0.4, 1.0, 4.0), (0.2, 0.4, 1.6))):
        kxyz = xyz[graph.nearest_point(xyz, graph.voxel_down_sample(xyz, voxel))]
        for lvl, (pts, ctr, r) in enumerate(((xyz, kxyz, r0), (kxyz, kxyz, r1))):
            e = graph.canonical_edges(ref.gen_disjointed_rnn_local_graph_v3(pts, ctr, r, -1))
            out['edges_%d_%d' % (i, lvl)] = e.astype(np.int32)
    np.savez_compressed(os.path.join(GOLDEN, 'graph_live_reference.npz'), **out)
    print('graph_live_reference:', {k: v.shape for k, v in out.items()})


def checkpoint_fixtures():
    """checkpoints/<cfg>/: the reference's `checkpoint` state file and model-N.index of every shipped checkpoint, and
    the gzipped model-N.meta of the two the saved-graph test re-interprets.  The tensor bytes are not stored: the
    data file is rebuilt from weights_<cfg>.npz (oracle/checkpoint_fixture.py), checked against the index's CRC32C."""
    import gzip
    import shutil
    from oracle import checkpoint_fixture
    root = os.path.join(reference_graph.REFERENCE_ROOT, 'checkpoints')
    for name in sorted(os.listdir(root)):
        dst = os.path.join(checkpoint_fixture.FIXTURES, name)
        os.makedirs(dst, exist_ok=True)
        for f in os.listdir(os.path.join(root, name)):
            path = os.path.join(root, name, f)
            if f == 'checkpoint' or f.endswith('.index'):
                shutil.copy(path, dst)
            elif f.endswith('.meta') and name in ('car_auto_T1_train', 'car_fixed_T3_train'):
                with open(path, 'rb') as i, gzip.GzipFile(os.path.join(dst, f + '.gz'), 'wb', mtime=0) as o:
                    o.write(i.read())
        tmp = tempfile.mkdtemp()
        try:
            checkpoint_fixture.rebuild(name, tmp)        # raises unless every tensor matches the index's CRC32C
        finally:
            shutil.rmtree(tmp)
        print('checkpoint fixture', name)


KITTI_EVAL_TREES = {   # name -> synthetic_tree arguments
    'mixed': dict(seed=31, num_frames=60, big_frames=(7,)),
    'no_aos_no_cyclist': dict(seed=32, num_frames=30, alpha_invalid=True, never_detected=(2,)),
}


def kitti_eval_goldens():
    """tests/golden/kitti_eval_<tree>.json: seeded synthetic label / result trees (oracle/kitti_eval.synthetic_tree)
    and everything the reference's own evaluator writes and prints on them - the binary oracle/kitti_eval_build.py
    compiles from kitti_native_evaluation/src/evaluate_object_3d_offline.cpp with the Boost stand-in.  The result
    file names skip index 3, and label file 000003.txt exists without a result file (it must not be evaluated)."""
    import subprocess
    from oracle import kitti_eval as ke
    from oracle import kitti_eval_build
    binary = kitti_eval_build.build()
    assert binary, 'needs the reference tree'
    for name, kw in KITTI_EVAL_TREES.items():
        gt_texts, det_texts = ke.synthetic_tree(**kw)
        names = ['%06d.txt' % (i if i < 3 else i + 1) for i in range(len(gt_texts))]
        tmp = tempfile.mkdtemp()
        gt_dir, res_dir = os.path.join(tmp, 'label_2'), os.path.join(tmp, 'results')
        ke.write_tree(gt_dir, res_dir, gt_texts, det_texts, names)
        with open(os.path.join(gt_dir, '000003.txt'), 'w') as f:
            f.write('Car 0.00 0 0.1 100 100 200 200 1.5 1.6 3.9 1.0 1.6 10.0 0.1\n')
        stdout = subprocess.run([binary, gt_dir, res_dir], capture_output=True, text=True, check=True).stdout
        outputs = {}
        for d, _, files in os.walk(res_dir):
            for fname in files:
                rel = os.path.relpath(os.path.join(d, fname), res_dir)
                if not rel.startswith('data' + os.sep):
                    with open(os.path.join(d, fname)) as f:
                        outputs[rel] = f.read()
        gts = {n: t for n, t in zip(names, gt_texts)}
        gts['000003.txt'] = open(os.path.join(gt_dir, '000003.txt')).read()
        with open(os.path.join(GOLDEN, 'kitti_eval_%s.json' % name), 'w') as f:
            json.dump({'tree': kw, 'label_2': gts, 'data': dict(zip(names, det_texts)), 'outputs': outputs,
                       'stdout': stdout}, f, indent=0, sort_keys=True)
        print('kitti_eval', name, 'frames', len(names), 'outputs', len(outputs))
        print(stdout)


BEAM_SEEDS, BEAM_POINTS = (41, 42, 43), 6000          # small frames: the reference script end to end
BEAM_FULL_SEEDS, BEAM_FULL_POINTS = (51, 52), 120000    # full-size frames: scikit-learn's inertia only


def beam_downsample_goldens():
    """tests/golden/beam_downsample.npz: the reference's OWN scripts/point_cloud_downsample.py, run unmodified through
    runpy from a temporary directory laid out as its hard-coded ``../dataset/kitti/...`` paths, on a synthetic
    training tree (oracle.kitti.write_synthetic_kitti) with a ``3DOP_splits/val.txt`` listing every frame.  Shims,
    none of which touches the arithmetic the fixture pins:
      * ``open3d`` is stubbed: the script imports it for its commented-out visualisation only;
      * ``np.bool = bool``: the alias NumPy 2 removed (the script's mask dtype);
      * ``sklearn.cluster.KMeans`` is wrapped: ``n_jobs`` (removed in scikit-learn 1.0) is dropped, and the fit
        uses ``n_init=10`` (the default of the scikit-learn of the reference's era) and ``random_state=0`` so the
        fixture can be regenerated; each fit's centres and inertia are recorded.
    Stored: each frame's velodyne rows, scikit-learn's centres (its own order) and inertia, and the bytes the
    script wrote.  Beside them, for two seeded full-size frames (oracle.beam_downsample.velodyne_frame, 120 000
    points), the same KMeans fit's inertia on the cosines and the SHA-256 of the frame's bytes."""
    import hashlib
    import runpy
    import shutil
    import types
    import sklearn.cluster
    from oracle import beam_downsample as obd
    from oracle import kitti as okitti
    fits = []
    real_kmeans = sklearn.cluster.KMeans

    class _KMeans(object):
        def __init__(self, n_clusters=8, n_jobs=None, **kwargs):
            self._km = real_kmeans(n_clusters=n_clusters, n_init=10, random_state=0, **kwargs)

        def fit(self, x):
            self._km.fit(x)
            self.cluster_centers_ = self._km.cluster_centers_
            self.inertia_ = self._km.inertia_
            fits.append((np.asarray(self.cluster_centers_, dtype=np.float64).reshape(-1), float(self.inertia_)))
            return self

    tmp = tempfile.mkdtemp()
    saved = (os.getcwd(), list(sys.path), sys.modules.get('open3d'), getattr(np, 'bool', None))
    try:
        root = os.path.join(tmp, 'dataset', 'kitti')
        names = okitti.write_synthetic_kitti(root, BEAM_SEEDS, num_points=BEAM_POINTS, test_split=False)
        os.makedirs(os.path.join(root, '3DOP_splits'))
        with open(os.path.join(root, '3DOP_splits', 'val.txt'), 'w') as f:
            f.write(''.join(n + '\n' for n in names))
        os.makedirs(os.path.join(tmp, 'scripts'))
        os.chdir(os.path.join(tmp, 'scripts'))
        sys.path.insert(0, reference_graph.REFERENCE_ROOT)
        sys.modules['open3d'] = types.ModuleType('open3d')
        np.bool = bool
        sklearn.cluster.KMeans = _KMeans
        runpy.run_path(os.path.join(reference_graph.REFERENCE_ROOT, 'scripts', 'point_cloud_downsample.py'),
                       run_name='__main__')
        out = {'names': np.array(names), 'downsample_rate': np.int64(2), 'num_clusters': np.int64(64)}
        assert len(fits) == len(names)
        for i, name in enumerate(names):
            velo = np.fromfile(os.path.join(root, 'velodyne', 'training', 'velodyne', name + '.bin'), dtype=np.float32)
            written = np.fromfile(os.path.join(root, 'velodyne', 'training_downsampled_2', 'velodyne', name + '.bin'),
                                  dtype=np.uint8)
            out['velo_%d' % i] = velo.reshape(-1, 4)
            out['bin_%d' % i] = written
            print('beam_downsample', name, 'points', len(velo) // 4, 'kept', len(written) // 16, 'inertia', fits[i][1])
        out['sk_centers'] = np.stack([c for c, _ in fits])
        out['sk_inertia'] = np.array([v for _, v in fits])
        del fits[:]
        sha, inertia = [], []
        for seed in BEAM_FULL_SEEDS:
            velo = obd.velodyne_frame(seed, BEAM_FULL_POINTS)
            sha.append(hashlib.sha256(velo.tobytes()).hexdigest())
            _KMeans(n_clusters=64, n_jobs=-1).fit(obd.cosines(velo[:, :3]).reshape(-1, 1))
            inertia.append(fits[-1][1])
            print('beam_downsample full-size seed', seed, 'inertia', inertia[-1])
        out['full_seeds'] = np.array(BEAM_FULL_SEEDS, dtype=np.int64)
        out['full_num_points'] = np.int64(BEAM_FULL_POINTS)
        out['full_sha256'] = np.array(sha)
        out['full_sk_inertia'] = np.array(inertia)
        np.savez_compressed(os.path.join(GOLDEN, 'beam_downsample.npz'), **out)
    finally:
        os.chdir(saved[0])
        sys.path[:] = saved[1]
        if saved[2] is None:
            sys.modules.pop('open3d', None)
        else:
            sys.modules['open3d'] = saved[2]
        if saved[3] is None and hasattr(np, 'bool'):
            del np.bool
        sklearn.cluster.KMeans = real_kmeans
        shutil.rmtree(tmp)


if __name__ == '__main__':
    which = sys.argv[1] if len(sys.argv) > 1 else 'all'
    if which in ('all', 'beam_downsample'):
        beam_downsample_goldens()
    if which in ('all', 'graph_random'):
        graph_random_goldens()
    if which in ('all', 'graph_multiscale'):
        graph_multiscale_goldens()
    if which in ('all', 'graph_scale'):
        graph_scale_goldens()
    if which in ('all', 'graph_rnd3d'):
        graph_rnd3d_goldens()
    if which in ('all', 'gnn'):
        main()
    if which in ('all', 'post'):
        post_goldens()
    if which in ('all', 'box_canonical'):
        box_canonical_goldens()
    if which in ('all', 'kitti'):
        kitti_goldens()
    if which in ('all', 'kitti_voxel_avg'):
        kitti_voxel_avg_goldens()
    if which in ('all', 'graph_live_reference'):
        graph_live_reference_goldens()
    if which in ('all', 'checkpoints'):
        checkpoint_fixtures()
    if which in ('all', 'kitti_eval'):
        kitti_eval_goldens()
