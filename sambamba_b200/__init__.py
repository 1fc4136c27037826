"""sambamba_b200 -- H100-native (sm_90a) engine behind `sambamba depth` (see DESIGN.md).

Python is only the test/bench harness around libbdepth.so (the C ABI in include/bdepth.h);
the product is the CUDA library and the C++ CLI host in sambamba_b200/csrc.
"""
from ._lib import BDepth, BDepthError, lib_path, load_library, nccl_unique_id, plan_region_chunks, plan_shards  # noqa: F401
