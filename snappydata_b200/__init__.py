"""snappydata_b200 -- H100-native (sm_90a) scan/decode/filter/partial-aggregate engine for
SnappyData's column-store read path (see DESIGN.md).

Only what the hot path needs lives here:

  csrc/            CUDA kernels (sm_90a) + the C-ABI shared library (libsnappygpu.so)
  column_format    host-side ColumnBatch byte-format writer/reader (the reference's
                   ColumnEncoding layouts), used to build fixtures and synthetic tables
  lineitem         synthetic TPC-H lineitem-shaped column tables (counter-based generator,
                   identical on host/numpy and on device)
  capi             ctypes binding of include/snappy_gpu.h
  plan             expression DSL that flattens to sd_plan_desc (what the Scala operators serialise)
  exchange         the one cross-partition exchange of partial results (torch.distributed plumbing)
  csrc/sd_operators.hpp   C++ mirror of the reference operator surface
                   (ColumnBatchIterator / SnappyHashAggregateExec / CollectAggregateExec)
"""

__version__ = "0.1.0"
