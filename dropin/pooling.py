"""Drop-in shim: `import pooling` resolves to the H100-native implementation
(put this directory first on sys.path instead of the reference checkout)."""
from fewshot_detection_b200.pooling import *  # noqa: F401,F403
