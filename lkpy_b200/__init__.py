"""
lkpy_b200 — H100-native engines for LensKit's two compute hot paths.

* ALS half-epoch (implicit / explicit), replacing ``src/accel/als/*.rs``
* item-kNN similarity build + neighbourhood scoring, replacing
  ``src/accel/knn/{item_train,item_score,accum}.rs``

The product path is hand-written sm_90a CUDA behind a C-ABI shared library
(``include/lkpy_b200.h`` → ``lkpy_b200/csrc/liblkpy_b200.so``).  There is no CPU
fallback: calling an engine entry point without the library or without a CUDA
device raises.  ``oracle/`` is test infrastructure only.
"""

__version__ = "0.1.0"
