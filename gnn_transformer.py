"""Drop-in for the reference's gnn_transformer.py: same names, CUDA (sm_90a) implementation."""
from fira_icse_b200.modules import (Attention, Combination, Decoder, Encoder, FeedForward, GCN,  # noqa: F401
                                    position_encoding)
