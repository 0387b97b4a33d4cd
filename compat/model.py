"""`from model import SAGEDeterministic` (reference pert_gnn.py:12) resolved to the H100 implementation.
Put this directory first on PYTHONPATH:  PYTHONPATH=/path/to/repo/compat:/path/to/repo python pert_gnn.py ..."""
from pert_gnn_kdd23_b200.model import SAGEDeterministic  # noqa: F401
