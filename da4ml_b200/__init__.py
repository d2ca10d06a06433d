"""da4ml_b200 -- GPU-native (sm_90a CUDA, H100) CMVM distributed-arithmetic solver.

Drop-in for the ``da4ml.cmvm.solve`` path of calad0i/da4ml; see DESIGN.md / INTEGRATION.md.
"""

__version__ = '0.1.0'
