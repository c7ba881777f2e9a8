"""polara_b200 -- H100-native (sm_90a) engine behind the Polara SVD/CoFFee model API.

Host code is Python; all computation happens in hand-written CUDA reached through the
C-ABI of ``libpolara_b200.so`` (see include/polara_b200.h).  No CPU fallback.
"""
__version__ = "0.1.0"
