"""Drop-in shim: `import utils` / `from utils import *` resolves to the H100-native implementation
(put this directory first on sys.path instead of the reference checkout)."""
from fewshot_detection_b200.utils import *  # noqa: F401,F403
from fewshot_detection_b200.utils import (bbox_iou, get_region_boxes, get_region_boxes_v2, nms, read_data_cfg,  # noqa: F401
                                          logging, region_detections, Detections, ImageDetections, get_image_size,
                                          load_class_names)
