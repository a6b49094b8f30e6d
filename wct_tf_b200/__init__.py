"""wct_tf_b200 -- H100-native (sm_90a) multi-level WCT stylisation engine (inference hot path of eridgd/WCT-TF)."""
__version__ = "0.1.0"

from .model import WCTModel, RELU_TARGETS_ALL  # noqa: F401


def __getattr__(name):  # lazy: importing the package must not need the CUDA library
    if name == "WCT":
        from .wct import WCT
        return WCT
    raise AttributeError(name)
