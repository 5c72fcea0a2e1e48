"""monorec_b200 -- H100-native (sm_90a) implementation of MonoRec's data-parallel hot path.

Only what the path needs lives here: `csrc/` (CUDA kernels + the C-ABI shared library) and the
Python host-side mirror of the reference interface (`CostVolumeModule`, `MaskModule`,
`DepthModule`, `MonoRecModel`; reference: model/monorec/monorec_model.py:132-729).
"""
__version__ = "0.1.0"


def __getattr__(name):
    # lazy: importing the package must not require torch/CUDA until a module is touched
    if name in ("MonoRecModel", "CostVolumeModule", "MaskModule", "DepthModule", "ResnetEncoder"):
        from . import model as _m
        return getattr(_m, name)
    if name in ("ResidualImage", "ResidualImageModule"):
        from . import layers as _l
        return getattr(_l, name)
    if name in ("RobotCarLidar", "lidar_depth"):
        from . import robotcar as _r
        return getattr(_r, name)
    raise AttributeError(name)
