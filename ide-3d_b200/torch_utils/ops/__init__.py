"""sm_90a implementations of the reference's torch_utils/ops package (same module and function names)."""
