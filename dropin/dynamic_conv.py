"""Drop-in shim: `import dynamic_conv` resolves to the H100-native implementation
(put this directory first on sys.path instead of the reference checkout)."""
from fewshot_detection_b200.dynamic_conv import *  # noqa: F401,F403
