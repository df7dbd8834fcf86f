"""Drop-in shim: `import cfg` resolves to the H100-native implementation
(put this directory first on sys.path instead of the reference checkout)."""
from fewshot_detection_b200.cfg import *  # noqa: F401,F403
from fewshot_detection_b200.cfg import cfg, parse_cfg, load_conv, load_conv_bn, save_conv, save_conv_bn  # noqa: F401
