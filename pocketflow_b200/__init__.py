"""pocketflow_b200 — H100-native compression-aware training step behind PocketFlow's
AbstractLearner / AbstractModelHelper plugin surface.  Compute lives in libpf_b200.so
(hand-written sm_90a CUDA, C ABI in include/pf_b200.h); there is no CPU fallback."""
__version__ = '0.1.0'
