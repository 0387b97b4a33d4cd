"""pert_gnn_kdd23_b200 -- H100-native hot path of PERT-GNN (see DESIGN.md)."""
__version__ = "0.1.0"
