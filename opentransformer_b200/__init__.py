"""opentransformer_b200 -- the OpenTransformer speech-transformer hot path as hand-written sm_90a
CUDA kernels behind the reference's nn.Module / Recognizer interface (see DESIGN.md)."""
from ._lib import LIB_PATH, exported_symbols  # noqa: F401

__all__ = ['LIB_PATH', 'exported_symbols']
