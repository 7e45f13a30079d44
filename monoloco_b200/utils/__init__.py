from .iou import calculate_iou, get_iou_matrix, get_iou_matches, reorder_matches
from .camera import pixel_to_camera, get_keypoints, xyz_from_distance
from .kitti import save_txts, kitti_rows
from .logs import set_logger
