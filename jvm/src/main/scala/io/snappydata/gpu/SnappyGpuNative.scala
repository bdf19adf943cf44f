/*
 * JVM binding of libsnappygpu.so (see include/snappy_gpu.h and jvm/native/snappy_gpu_jni.c).
 * NOT COMPILED in this repository's container (no JDK/Scala toolchain); written against SnappyData 1.3.0 /
 * snappy-spark 2.1.1.9 class names as they appear in /root/reference.  The natives follow the only native precedent of
 * the reference, org.apache.spark.unsafe.Native (aqp/src/main/cpp/io/snappydata/DataOptimizations.c:26-68): raw
 * addresses and sizes, primitive returns; a non-zero sd_status becomes RuntimeException(sd_last_error()).
 */
package io.snappydata.gpu

object SnappyGpuNative {
  // loaded opportunistically like org.apache.spark.unsafe.Native
  // (cluster/src/test/scala/org/apache/spark/unsafe/NativeUTF8StringPropertyCheckSuite.scala:58)
  lazy val isLoaded: Boolean = try {
    System.loadLibrary("snappygpujni"); true
  } catch { case _: UnsatisfiedLinkError => false }

  @native def init(device: Int): Int
  @native def planCreate(planDescAddr: Long): Long
  @native def planSetLiterals(plan: Long, literalsAddr: Long, n: Int): Unit
  /** per column either a native address (direct ByteBuffer) or a heap byte[] + offset (copied by the shim into its
    * page-locked staging area: no array is pinned while CUDA work is queued) */
  @native def batchSubmit(plan: Long, numRows: Int, nCols: Int,
      colAddrs: Array[Long], colLens: Array[Long], heapCols: Array[Array[Byte]], heapOffsets: Array[Int],
      delta0Addrs: Array[Long], delta0Lens: Array[Long], delta0Heap: Array[Array[Byte]], delta0Offsets: Array[Int],
      delta1Addrs: Array[Long], delta1Lens: Array[Long], delta1Heap: Array[Array[Byte]], delta1Offsets: Array[Int],
      deleteAddr: Long, deleteLen: Long, deleteHeap: Array[Byte], deleteOffset: Int,
      statsAddr: Long, statsLen: Long, statsHeap: Array[Byte], statsOffset: Int, statsNCols: Int,
      bucketId: Int, batchId: Long): Unit
  @native def rowsSubmit(plan: Long, rowsAddr: Long, len: Long, nrows: Int): Unit
  /** bytes written to outAddr; -needed when cap is too small (the execution is complete, call again) */
  @native def planFinish(plan: Long, outAddr: Long, cap: Long): Long
  @native def planReset(plan: Long): Unit
  @native def planMetrics(plan: Long, out: Array[Long]): Unit
  @native def planDestroy(plan: Long): Unit
  @native def finalMerge(planDescAddr: Long, rowsAddr: Long, len: Long, outAddr: Long, cap: Long): Long

  // ---- residency (INTEGRATION.md 4): a server keeps the ColumnBatches of its buckets in HBM across queries --------------
  /** schemaAddr: nCols x sd_column (layout pinned in jvm/abi_offsets.txt), written by GpuPlanSerializer */
  @native def storeCreate(device: Int, nCols: Int, schemaAddr: Long): Long
  /** same buffer conventions as batchSubmit; the batch is resident when the call returns */
  @native def storePutBatch(store: Long, numRows: Int, nCols: Int,
      colAddrs: Array[Long], colLens: Array[Long], heapCols: Array[Array[Byte]], heapOffsets: Array[Int],
      delta0Addrs: Array[Long], delta0Lens: Array[Long], delta0Heap: Array[Array[Byte]], delta0Offsets: Array[Int],
      delta1Addrs: Array[Long], delta1Lens: Array[Long], delta1Heap: Array[Array[Byte]], delta1Offsets: Array[Int],
      deleteAddr: Long, deleteLen: Long, deleteHeap: Array[Byte], deleteOffset: Int,
      statsAddr: Long, statsLen: Long, statsHeap: Array[Byte], statsOffset: Int, statsNCols: Int,
      bucketId: Int, batchId: Long): Unit
  @native def storeDestroy(store: Long): Unit
  /** scan the resident batches of these buckets (null: all) with the literals set by planSetLiterals; a store that has
    * grown since the plan's last scan is re-scanned incrementally (only the new batches get descriptors) */
  @native def planScanStore(plan: Long, store: Long, bucketIds: Array[Int]): Unit
  /** UPDATE of the resident batches (ColumnUpdateExec): plan built with SD_PLAN_MUTATE, targetCols(i) = table ordinal that
    * the plan's i-th projection writes, literals = sd_literal array at literalsAddr; returns the rows updated */
  @native def planUpdateStore(plan: Long, store: Long, bucketIds: Array[Int], literalsAddr: Long, nLiterals: Int,
      targetCols: Array[Int]): Long
  /** DELETE of the resident rows the plan's filter matches (ColumnDeleteExec); returns the rows deleted */
  @native def planDeleteStore(plan: Long, store: Long, bucketIds: Array[Int], literalsAddr: Long, nLiterals: Int): Long
  /** folds update deltas and delete masks of the store's dirty batches (bucketIds null = all) back into their base columns;
    * batches with (deleted rows + delta entries) >= minDirtyFraction * rows are rewritten, fully deleted ones removed.
    * out(0) batches rewritten, out(1) removed, out(2) deleted rows purged, out(3) bytes written.  Rewritten batches number
    * their live rows from 0: later UPDATE / DELETE positions and any JVM-side mirror of the bytes follow the new version */
  @native def compactStore(store: Long, bucketIds: Array[Int], minDirtyFraction: Double, out: Array[Long]): Unit
  /** gives back the device memory of superseded batch versions; call it after a compaction.  Slabs at most
    * maxLiveFraction live are emptied into fresh ones first (0: only dead slabs are freed, 1: everything is repacked).
    * A scan pins what it may read until its plan finishes, is reset or destroyed: such slabs are deferred to a later call.
    * out(0) slabs freed, out(1) slab bytes freed, out(2) bytes copied, out(3) slabs deferred */
  @native def reclaimStore(store: Long, maxLiveFraction: Double, out: Array[Long]): Unit

  // ---- the exchange between co-located GPU partitions (INTEGRATION.md 4b) ------------------------------------------------
  /** rank 0 calls this and broadcasts the 128 bytes; every rank passes them to commCreate */
  @native def commUniqueId(out128: Array[Byte]): Unit
  /** blocks until all `world` ranks have joined */
  @native def commCreate(id128: Array[Byte], rank: Int, world: Int, device: Int): Long
  @native def commDestroy(comm: Long): Unit
  /** after this partition's scans: all-gather + merge; planFinish then returns the merged partial rows on every rank */
  @native def planExchange(plan: Long, comm: Long): Unit

  // ---- page-locked host memory --------------------------------------------------------------------------------------------
  /** for planFinish's output (the projected rows of a scan without aggregate arrive in ONE device->host copy at link speed
    * when the buffer is page-locked) and for long-lived staging; wrap with Platform.* / UnsafeRow.pointTo(null, addr, size) */
  @native def hostAlloc(bytes: Long): Long
  @native def hostFree(addr: Long): Unit
}
