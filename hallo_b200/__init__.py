"""hallo_b200: H100-native (sm_90a) implementation of the Hallo denoising hot path."""
__version__ = "0.1.0"
