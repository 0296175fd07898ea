"""Drop-in for the reference's Model.py: same names, CUDA (sm_90a) implementation."""
from fira_icse_b200.model import CopyNet, TransModel  # noqa: F401
