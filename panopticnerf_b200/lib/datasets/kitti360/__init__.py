"""KITTI-360 on-disk formats in front of the render path (SURVEY 8(f) rank 3): calibration and pose text files,
the fisheye (MEI) yaml, the 3D bounding-box annotation XML -> the primitive table the renderer consumes, an
intersection cache, the frames of a sequence as a device FrameSet for training batches (frames.py), and their depth
targets projected from the sequence's Velodyne scans (lidar.py) or matched from its stereo pair (stereo.py), and the
camera masks of weighted training draws (masks.py).  The
reference's dataset code is not in the mount; the formats follow the public KITTI-360 documentation / kitti360scripts
as recalled, every reader says what it expects and fails loudly on anything else."""
from .calib import (load_cam0_to_world, load_cam_to_pose, load_fisheye_yaml, load_perspective, load_poses,
                    perspective_batch, fisheye_batch)
from .bboxes import Box3D, boxes_to_primitives, parse_bboxes_xml, primitive_batch, sequence_primitives
from .intersection_cache import load_intersections, save_intersections
from .groundtruth import load_panoptic_gt, load_semantic_gt
from .frames import load_frames
from .lidar import lidar_depth, load_cam_to_velo, load_velodyne, save_depth_png
from .stereo import stereo_depth, stereo_disparity
from .masks import fisheye_fov_mask, load_camera_mask

__all__ = ["load_cam0_to_world", "load_cam_to_pose", "load_fisheye_yaml", "load_perspective", "load_poses",
           "perspective_batch", "fisheye_batch", "Box3D", "boxes_to_primitives", "parse_bboxes_xml",
           "primitive_batch", "sequence_primitives", "load_intersections", "save_intersections", "load_panoptic_gt", "load_semantic_gt",
           "load_frames", "lidar_depth", "load_cam_to_velo", "load_velodyne", "save_depth_png",
           "stereo_depth", "stereo_disparity", "fisheye_fov_mask", "load_camera_mask"]
