"""KITTI-360 on-disk formats in front of the render path (SURVEY 8(f) rank 3): calibration and pose text files,
the fisheye (MEI) yaml, the 3D bounding-box annotation XML -> the primitive table the renderer consumes, and an
intersection cache.  The reference's dataset code is not in the mount; the formats follow the public KITTI-360
documentation / kitti360scripts as recalled, every reader says what it expects and fails loudly on anything else."""
from .calib import (load_cam0_to_world, load_cam_to_pose, load_fisheye_yaml, load_perspective, load_poses,
                    perspective_batch, fisheye_batch)
from .bboxes import Box3D, boxes_to_primitives, parse_bboxes_xml, primitive_batch
from .intersection_cache import load_intersections, save_intersections
from .groundtruth import load_panoptic_gt, load_semantic_gt

__all__ = ["load_cam0_to_world", "load_cam_to_pose", "load_fisheye_yaml", "load_perspective", "load_poses",
           "perspective_batch", "fisheye_batch", "Box3D", "boxes_to_primitives", "parse_bboxes_xml",
           "primitive_batch", "load_intersections", "save_intersections", "load_panoptic_gt", "load_semantic_gt"]
