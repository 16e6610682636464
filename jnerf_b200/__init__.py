"""jnerf_b200: an H100-native (sm_90a) Instant-NGP inner loop behind JNeRF's plugin API.
The CUDA library is built by `jnerf_b200/build.py` (or __graft_entry__.build()); nothing here runs on the CPU."""
__version__ = "0.1.0"
