"""quickwit_b200 — H100-native drop-in for Quickwit's per-split leaf search hot path.

Layout (only what the path needs, see DESIGN.md):
  csrc/        CUDA kernels (sm_90a) + C++ host side + the C ABI (include/qwgpu.h) -> libqwgpu.so
  ffi.py       ctypes binding of the C ABI (no logic)
  service.py   host-side mirror of the reference interface: SearchService.leaf_search,
               LambdaLeafSearchInvoker.invoke_leaf_search, root-side merge
  proto.py     wire codec for the search.proto messages this path exchanges
  plan.py      seam-C plan construction helpers
  splitgen.py  split-image construction (documents / synthetic corpus) — not on the query path
"""
__version__ = "0.1.0"
