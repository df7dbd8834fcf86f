"""Drop-in shim: `import darknet_meta` resolves to the H100-native implementation
(put this directory first on sys.path instead of the reference checkout)."""
from fewshot_detection_b200.darknet_meta import *  # noqa: F401,F403
from fewshot_detection_b200.darknet_meta import Darknet  # noqa: F401
