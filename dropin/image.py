"""Drop-in shim: `import image` / `from image import *` resolves to the H100-native implementation
(put this directory first on sys.path instead of the reference checkout)."""
from fewshot_detection_b200.image import *  # noqa: F401,F403
from fewshot_detection_b200.image import (data_augmentation, fill_truth_detection, fill_truth_detection_meta,  # noqa: F401
                                          load_label, load_data_detection, load_data_with_label, rand_scale)
