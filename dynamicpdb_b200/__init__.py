"""dynamicpdb_b200: H100-native (sm_90a) DFOLDv2 score-network hot path (see DESIGN.md)."""
__version__ = "0.1.0"
