"""fewshot_detection_b200: the meta-training hot path of bingykang/Fewshot_Detection
(Darknet(cfg).forward / RegionLoss) on hand-written sm_90a CUDA kernels.

Importing the compute modules requires the in-tree `libfsdet.so`
(`python -c "import __graft_entry__ as g; g.build()"`); there is no CPU or
library fallback.  `fewshot_detection_b200.netcfg` and `.cfg` are importable
without it.
"""
__version__ = '0.1.0'

__all__ = ['cfg', 'netcfg']
