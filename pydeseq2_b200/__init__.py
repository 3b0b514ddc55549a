"""pydeseq2_b200 -- H100-native backend for PyDESeq2's per-gene NB-GLM hot path."""
__version__ = "0.1.0"


def __getattr__(name):  # lazy: importing the package must not require the CUDA library
    if name == "B200Inference":
        from .inference import B200Inference

        return B200Inference
    raise AttributeError(name)
