"""Drop-in shim: `import darknet` resolves to the H100-native implementation
(put this directory first on sys.path instead of the reference checkout)."""
from fewshot_detection_b200.darknet import *  # noqa: F401,F403
from fewshot_detection_b200.darknet import Darknet  # noqa: F401
