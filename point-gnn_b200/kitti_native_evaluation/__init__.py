"""KITTI object evaluation: the twin of the reference's kitti_native_evaluation/ (evaluate_object_3d_offline)."""
