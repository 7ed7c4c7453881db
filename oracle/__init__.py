"""CPU oracle for the Point-GNN per-frame message-passing hot path.

TEST INFRASTRUCTURE ONLY.  This package restates, on the CPU, the algorithm of
the reference files /root/reference/models/graph_gen.py, models/gnn.py and
models/models.py::predict.  Only ``tests/``, ``__graft_entry__.smoke()`` and
``bench.py``'s cpu_baseline / ``--impl reference`` leg may import it - and there
only as the checker / the timed CPU baseline, never as part of the product path
(``point-gnn_b200`` never imports ``oracle`` and fails loudly when the CUDA
library is missing).

Parity pinning (SURVEY.md section 8c): the reference ships NO golden vectors for
this path, so both halves are pinned against the reference ITSELF, executed in the
build container, with the fixtures and the generating script committed
(tests/golden/, tools/make_golden.py):

* graph half - the reference's own ``models/graph_gen.py`` (scikit-learn present)
  produces the edge lists of tests/golden/graph_*.npz;
* GNN half - the reference's own saved TensorFlow graph
  (checkpoints/<cfg>/model-N.meta, the MetaGraphDef train.py wrote) is decoded and
  interpreted node by node by ``oracle/graphdef.py`` (NumPy; TensorFlow itself
  cannot be installed) with the trained weights -> tests/golden/gnn_*.npz for all
  seven shipped checkpoints.  ``oracle/gnn.py`` reproduces those vectors exactly
  (tests/test_graphdef_cpu.py), so it is a checked restatement, not a guess.  The
  vectors pin what the shipped configs run: ReLU, the segment max, fp32.  The other
  activations and aggregations of the reference's table, and the library's FP16
  arithmetic, are arguments of the same functions, so they share that structure.

What remains a definition rather than a verified fact: Open3D 0.7's
``voxel_down_sample`` (binary package, source absent) - see oracle/graph.py.
"""
