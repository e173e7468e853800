"""Native extension packages of the CUDA backend (mirrors ``src/extensions_ref``)."""
