"""Drop-in shim: `import region_loss` resolves to the H100-native implementation
(put this directory first on sys.path instead of the reference checkout)."""
from fewshot_detection_b200.region_loss import *  # noqa: F401,F403
from fewshot_detection_b200.region_loss import RegionLoss, RegionLossV2, build_targets, neg_filter  # noqa: F401
