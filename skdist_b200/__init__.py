"""skdist_b200 -- H100-native engine behind the ``skdist.distribute`` API.

Host code (this package) mirrors the reference's meta-estimators; all fits run in
hand-written sm_90a CUDA kernels reached through the C-ABI of
``lib/libskdist_b200.so`` (see include/skdist_b200.h).  No CPU fallback.
"""
__version__ = "0.1.0"
