"""fira_icse_b200 -- H100-native (sm_90a) hot path of FIRA behind the reference's nn.Module surface.

The directory is `fira_icse_b200` (an importable identifier) for the package the task text calls
`fira-icse_b200`.  Importing the package does not need a GPU; running anything does, and fails
loudly when libfira_b200.so is missing -- there is no CPU fallback.
"""
from ._lib import FiraLibraryError, LIB_PATH  # noqa: F401
from .graph import PackedEdges  # noqa: F401
from .model import CopyNet, TransModel  # noqa: F401
from .optim import FlatAdam  # noqa: F401
from .modules import (Attention, Combination, CombinationLayer, Decoder, Encoder, FeedForward, GCN,  # noqa: F401
                      position_encoding)

__version__ = "0.1.0"
