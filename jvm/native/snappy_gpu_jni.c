/*
 * snappy_gpu_jni.c -- JNI shim between the reference's JVM operators and libsnappygpu.so.
 *
 * NOT COMPILED IN THIS REPOSITORY'S CONTAINER (no JDK here); `gcc -fsyntax-only -Ijvm/native/mock` checks it against a
 * minimal stand-in for <jni.h> (tests/test_jni_syntax.py).  Kept to the thin pattern of the reference's only native
 * precedent, org.apache.spark.unsafe.Native (/root/reference/aqp/src/main/cpp/io/snappydata/DataOptimizations.c:26-68):
 * static natives taking raw addresses and sizes as jlong/jint, returning primitives.
 *
 * Heap buffers.  Column buffers may be heap ByteBuffers (ColumnTableScan.scala:430-437 handles both kinds).  Their
 * bytes are COPIED with GetByteArrayRegion into a per-thread page-locked staging area (sd_host_alloc) before anything
 * else happens: no Get*Critical section is ever open (the JNI specification forbids other JNI calls, and blocking, inside
 * one), nothing of the Java heap is pinned while CUDA copies are queued, and the copies out of the staging area are
 * asynchronous DMA.  sd_batch_submit has consumed the staging area when it returns (default ownership rule,
 * ColumnBatchIterator.scala:165-184), so the next call reuses it.
 *
 * Build on a box with a JDK:
 *   gcc -O2 -shared -fPIC -I$JAVA_HOME/include -I$JAVA_HOME/include/linux -I../../include \
 *       snappy_gpu_jni.c -L../../snappydata_b200/csrc -lsnappygpu -o libsnappygpujni.so
 *
 * Scala side: jvm/src/main/scala/io/snappydata/gpu/SnappyGpuNative.scala.
 * Errors: non-zero sd_status -> RuntimeException(sd_last_error()); there is no CPU fallback.
 */
#include <jni.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "snappy_gpu.h"

#define JFN(name) Java_io_snappydata_gpu_SnappyGpuNative_00024_##name

static void throw_msg(JNIEnv* env, const char* cls_name, const char* msg) {
  if ((*env)->ExceptionCheck(env)) return;                 /* keep the first exception */
  jclass cls = (*env)->FindClass(env, cls_name);
  if (cls == NULL) return;                                 /* FindClass has raised NoClassDefFoundError */
  (*env)->ThrowNew(env, cls, msg ? msg : "libsnappygpu error");
}
static void throw_last(JNIEnv* env) { throw_msg(env, "java/lang/RuntimeException", sd_last_error()); }

/* ---- per-thread page-locked staging for heap byte[]s ---------------------------------------------------------- */
static __thread uint8_t* t_stage = NULL;
static __thread int64_t t_stage_cap = 0;
static __thread int64_t t_stage_used = 0;

static int stage_reserve(JNIEnv* env, int64_t total) {
  if (total <= t_stage_cap) return 0;
  int64_t cap = t_stage_cap ? t_stage_cap : (int64_t)32 << 20;
  while (cap < total) cap *= 2;
  void* p = NULL;
  if (sd_host_alloc(cap, &p)) { throw_last(env); return -1; }
  if (t_stage) sd_host_free(t_stage);
  t_stage = (uint8_t*)p; t_stage_cap = cap;
  return 0;
}
/* copy `len` bytes of `arr` starting at `off` into the staging area; returns the native address (NULL + exception on error) */
static const void* stage_bytes(JNIEnv* env, jbyteArray arr, jint off, jlong len) {
  if (arr == NULL) { throw_msg(env, "java/lang/NullPointerException", "heap column buffer is null"); return NULL; }
  if (off < 0 || len < 0 || (jlong)off + len > (jlong)(*env)->GetArrayLength(env, arr)) {
    throw_msg(env, "java/lang/ArrayIndexOutOfBoundsException", "heap column buffer: offset + length beyond the array");
    return NULL;
  }
  uint8_t* dst = t_stage + t_stage_used;
  (*env)->GetByteArrayRegion(env, arr, off, (jsize)len, (jbyte*)dst);
  if ((*env)->ExceptionCheck(env)) return NULL;
  t_stage_used += (len + 63) & ~(int64_t)63;
  return dst;
}

JNIEXPORT jint JNICALL JFN(init)(JNIEnv* env, jobject self, jint device) {
  (void)self;
  int rc = sd_init(device);
  if (rc) throw_last(env);
  return rc;
}

/* planDesc: address of a serialized sd_plan_desc built off-heap by GpuPlanSerializer (all pointers inside are absolute
 * addresses into the same off-heap block) */
JNIEXPORT jlong JNICALL JFN(planCreate)(JNIEnv* env, jobject self, jlong planDescAddr) {
  (void)self;
  sd_plan* p = NULL;
  if (sd_plan_create((const sd_plan_desc*)(intptr_t)planDescAddr, &p)) { throw_last(env); return 0; }
  return (jlong)(intptr_t)p;
}

JNIEXPORT void JNICALL JFN(planSetLiterals)(JNIEnv* env, jobject self, jlong plan, jlong literalsAddr, jint n) {
  (void)self;
  if (sd_plan_set_literals((sd_plan*)(intptr_t)plan, (const sd_literal*)(intptr_t)literalsAddr, n)) throw_last(env);
}

enum { MAXC = 256 };

/* one family of per-column buffers: native addresses (direct ByteBuffers) or heap byte[] + offset */
typedef struct col_family { jlong* addr; jlong* len; jobjectArray heap; jint* off; } col_family;

static int64_t family_heap_bytes(JNIEnv* env, const col_family* f, int n) {
  int64_t total = 0;
  if (f->addr == NULL || f->heap == NULL) return 0;
  for (int i = 0; i < n; i++)
    if (f->addr[i] == 0 && f->len[i] > 0) total += (f->len[i] + 63) & ~(int64_t)63;
  (void)env;
  return total;
}
/* fill out[i] / out_len[i]; returns -1 with a pending exception on error */
static int family_resolve(JNIEnv* env, const col_family* f, int n, const void** out, int64_t* out_len) {
  for (int i = 0; i < n; i++) {
    out[i] = NULL; out_len[i] = 0;
    if (f->addr == NULL) continue;
    out_len[i] = f->len[i];
    if (f->addr[i] != 0) { out[i] = (const void*)(intptr_t)f->addr[i]; continue; }   /* direct buffer */
    if (f->len[i] <= 0 || f->heap == NULL) continue;                                   /* absent */
    jbyteArray arr = (jbyteArray)(*env)->GetObjectArrayElement(env, f->heap, i);
    if ((*env)->ExceptionCheck(env)) return -1;
    out[i] = stage_bytes(env, arr, f->off ? f->off[i] : 0, f->len[i]);
    if (arr) (*env)->DeleteLocalRef(env, arr);
    if (out[i] == NULL) return -1;
  }
  return 0;
}

/* One ColumnBatch from the JVM -> sd_batch -> sd_batch_submit (to_store == 0: `handle` is an sd_plan) or sd_store_put_batch
 * (to_store != 0: `handle` is an sd_store; the batch becomes resident). */
static void do_batch(JNIEnv* env, int to_store, jlong handle, jint numRows, jint nCols,
    jlongArray colAddrs, jlongArray colLens, jobjectArray heapCols, jintArray heapOffsets,
    jlongArray delta0Addrs, jlongArray delta0Lens, jobjectArray delta0Heap, jintArray delta0Offsets,
    jlongArray delta1Addrs, jlongArray delta1Lens, jobjectArray delta1Heap, jintArray delta1Offsets,
    jlong deleteAddr, jlong deleteLen, jbyteArray deleteHeap, jint deleteOffset,
    jlong statsAddr, jlong statsLen, jbyteArray statsHeap, jint statsOffset, jint statsNCols,
    jint bucketId, jlong batchId) {
  const void* cols[MAXC]; const void* d0[MAXC]; const void* d1[MAXC];
  int64_t lens[MAXC], d0l[MAXC], d1l[MAXC];
  if (nCols < 0 || nCols > MAXC) { throw_msg(env, "java/lang/IllegalArgumentException", "batchSubmit: 0 <= nCols <= 256"); return; }
  if (colAddrs == NULL || colLens == NULL) { throw_msg(env, "java/lang/NullPointerException", "batchSubmit: column arrays"); return; }
  col_family fc = {NULL, NULL, heapCols, NULL}, f0 = {NULL, NULL, delta0Heap, NULL}, f1 = {NULL, NULL, delta1Heap, NULL};
  int rc = -1, ok = 0;
  /* plain (non-critical) element access: copies or pins at the VM's discretion, JNI calls stay legal */
  fc.addr = (*env)->GetLongArrayElements(env, colAddrs, NULL);
  fc.len = (*env)->GetLongArrayElements(env, colLens, NULL);
  fc.off = heapOffsets ? (*env)->GetIntArrayElements(env, heapOffsets, NULL) : NULL;
  if (delta0Addrs && delta0Lens) {
    f0.addr = (*env)->GetLongArrayElements(env, delta0Addrs, NULL);
    f0.len = (*env)->GetLongArrayElements(env, delta0Lens, NULL);
    f0.off = delta0Offsets ? (*env)->GetIntArrayElements(env, delta0Offsets, NULL) : NULL;
  }
  if (delta1Addrs && delta1Lens) {
    f1.addr = (*env)->GetLongArrayElements(env, delta1Addrs, NULL);
    f1.len = (*env)->GetLongArrayElements(env, delta1Lens, NULL);
    f1.off = delta1Offsets ? (*env)->GetIntArrayElements(env, delta1Offsets, NULL) : NULL;
  }
  if (fc.addr == NULL || fc.len == NULL || (delta0Addrs && (f0.addr == NULL || f0.len == NULL)) ||
      (delta1Addrs && (f1.addr == NULL || f1.len == NULL))) goto done;          /* OutOfMemoryError is pending */
  {
    int64_t need = family_heap_bytes(env, &fc, nCols) + family_heap_bytes(env, &f0, nCols) + family_heap_bytes(env, &f1, nCols);
    if (deleteAddr == 0 && deleteHeap != NULL && deleteLen > 0) need += (deleteLen + 63) & ~(int64_t)63;
    if (statsAddr == 0 && statsHeap != NULL && statsLen > 0) need += (statsLen + 63) & ~(int64_t)63;
    t_stage_used = 0;
    if (stage_reserve(env, need)) goto done;
  }
  if (family_resolve(env, &fc, nCols, cols, lens) || family_resolve(env, &f0, nCols, d0, d0l) ||
      family_resolve(env, &f1, nCols, d1, d1l)) goto done;
  {
    sd_batch b;
    memset(&b, 0, sizeof(b));
    b.num_rows = numRows; b.ncols = nCols; b.col_bufs = cols; b.col_lens = lens;
    b.delta0 = f0.addr ? d0 : NULL; b.delta0_lens = d0l; b.delta1 = f1.addr ? d1 : NULL; b.delta1_lens = d1l;
    if (deleteAddr != 0) b.delete_buf = (const void*)(intptr_t)deleteAddr;
    else if (deleteHeap != NULL && deleteLen > 0) { b.delete_buf = stage_bytes(env, deleteHeap, deleteOffset, deleteLen); if (!b.delete_buf) goto done; }
    b.delete_len = b.delete_buf ? deleteLen : 0;
    if (statsAddr != 0) b.stats_row = (const void*)(intptr_t)statsAddr;
    else if (statsHeap != NULL && statsLen > 0) { b.stats_row = stage_bytes(env, statsHeap, statsOffset, statsLen); if (!b.stats_row) goto done; }
    b.stats_len = b.stats_row ? statsLen : 0;
    b.stats_ncols = statsNCols; b.bucket_id = bucketId; b.batch_id = batchId;
    /* every Java array has been copied or is a direct buffer retained by the iterator: nothing is pinned from here on */
    rc = to_store ? sd_store_put_batch((sd_store*)(intptr_t)handle, &b) : sd_batch_submit((sd_plan*)(intptr_t)handle, &b);
    ok = 1;
  }
done:
  if (fc.addr) (*env)->ReleaseLongArrayElements(env, colAddrs, fc.addr, JNI_ABORT);
  if (fc.len) (*env)->ReleaseLongArrayElements(env, colLens, fc.len, JNI_ABORT);
  if (fc.off) (*env)->ReleaseIntArrayElements(env, heapOffsets, fc.off, JNI_ABORT);
  if (f0.addr) (*env)->ReleaseLongArrayElements(env, delta0Addrs, f0.addr, JNI_ABORT);
  if (f0.len) (*env)->ReleaseLongArrayElements(env, delta0Lens, f0.len, JNI_ABORT);
  if (f0.off) (*env)->ReleaseIntArrayElements(env, delta0Offsets, f0.off, JNI_ABORT);
  if (f1.addr) (*env)->ReleaseLongArrayElements(env, delta1Addrs, f1.addr, JNI_ABORT);
  if (f1.len) (*env)->ReleaseLongArrayElements(env, delta1Lens, f1.len, JNI_ABORT);
  if (f1.off) (*env)->ReleaseIntArrayElements(env, delta1Offsets, f1.off, JNI_ABORT);
  if (ok && rc) throw_last(env);
}

#define BATCH_PARAMS jint numRows, jint nCols, \
    jlongArray colAddrs, jlongArray colLens, jobjectArray heapCols, jintArray heapOffsets, \
    jlongArray delta0Addrs, jlongArray delta0Lens, jobjectArray delta0Heap, jintArray delta0Offsets, \
    jlongArray delta1Addrs, jlongArray delta1Lens, jobjectArray delta1Heap, jintArray delta1Offsets, \
    jlong deleteAddr, jlong deleteLen, jbyteArray deleteHeap, jint deleteOffset, \
    jlong statsAddr, jlong statsLen, jbyteArray statsHeap, jint statsOffset, jint statsNCols, jint bucketId, jlong batchId
#define BATCH_ARGS numRows, nCols, colAddrs, colLens, heapCols, heapOffsets, delta0Addrs, delta0Lens, delta0Heap, delta0Offsets, \
    delta1Addrs, delta1Lens, delta1Heap, delta1Offsets, deleteAddr, deleteLen, deleteHeap, deleteOffset, \
    statsAddr, statsLen, statsHeap, statsOffset, statsNCols, bucketId, batchId

JNIEXPORT void JNICALL JFN(batchSubmit)(JNIEnv* env, jobject self, jlong plan, BATCH_PARAMS) {
  (void)self;
  do_batch(env, 0, plan, BATCH_ARGS);
}

/* ---- residency (INTEGRATION.md section 4): batches kept in HBM across queries ------------------------------------- */
/* schemaAddr: nCols x sd_column (type, nullable, table_ordinal, scale, precision: jvm/abi_offsets.txt) */
JNIEXPORT jlong JNICALL JFN(storeCreate)(JNIEnv* env, jobject self, jint device, jint nCols, jlong schemaAddr) {
  (void)self;
  sd_store* s = NULL;
  if (sd_store_create(device, nCols, (const sd_column*)(intptr_t)schemaAddr, &s)) { throw_last(env); return 0; }
  return (jlong)(intptr_t)s;
}
JNIEXPORT void JNICALL JFN(storePutBatch)(JNIEnv* env, jobject self, jlong store, BATCH_PARAMS) {
  (void)self;
  do_batch(env, 1, store, BATCH_ARGS);
}
JNIEXPORT void JNICALL JFN(storeDestroy)(JNIEnv* env, jobject self, jlong store) {
  (void)env; (void)self;
  sd_store_destroy((sd_store*)(intptr_t)store);
}
/* scan the resident batches of `bucketIds` (all buckets when null) with the plan's current literals */
JNIEXPORT void JNICALL JFN(planScanStore)(JNIEnv* env, jobject self, jlong plan, jlong store, jintArray bucketIds) {
  (void)self;
  jint* ids = NULL;
  jsize n = 0;
  if (bucketIds != NULL) {
    n = (*env)->GetArrayLength(env, bucketIds);
    ids = (*env)->GetIntArrayElements(env, bucketIds, NULL);
    if (ids == NULL) return;                                 /* OutOfMemoryError is pending */
  }
  int rc = sd_plan_scan_store((sd_plan*)(intptr_t)plan, (sd_store*)(intptr_t)store, (const int32_t*)ids, (int32_t)n);
  if (ids) (*env)->ReleaseIntArrayElements(env, bucketIds, ids, JNI_ABORT);
  if (rc) throw_last(env);
}

/* ColumnUpdateExec / ColumnDeleteExec hand their statement over here: the WHERE and SET expressions are the plan's, the literal
 * values an sd_literal array at literalsAddr (same layout as planSetLiterals); returns the number of rows changed */
JNIEXPORT jlong JNICALL JFN(planUpdateStore)(JNIEnv* env, jobject self, jlong plan, jlong store, jintArray bucketIds,
                                             jlong literalsAddr, jint nLiterals, jintArray targetCols) {
  (void)self;
  jint* ids = NULL;
  jsize n = 0;
  if (bucketIds != NULL) {
    n = (*env)->GetArrayLength(env, bucketIds);
    ids = (*env)->GetIntArrayElements(env, bucketIds, NULL);
    if (ids == NULL) return 0;                               /* OutOfMemoryError is pending */
  }
  jint* tc = (*env)->GetIntArrayElements(env, targetCols, NULL);
  if (tc == NULL) { if (ids) (*env)->ReleaseIntArrayElements(env, bucketIds, ids, JNI_ABORT); return 0; }
  int64_t rows = 0;
  int rc = sd_plan_update_store((sd_plan*)(intptr_t)plan, (sd_store*)(intptr_t)store, (const int32_t*)ids, (int32_t)n,
                                (const sd_literal*)(intptr_t)literalsAddr, nLiterals, (const int32_t*)tc, &rows);
  (*env)->ReleaseIntArrayElements(env, targetCols, tc, JNI_ABORT);
  if (ids) (*env)->ReleaseIntArrayElements(env, bucketIds, ids, JNI_ABORT);
  if (rc) throw_last(env);
  return (jlong)rows;
}

JNIEXPORT jlong JNICALL JFN(planDeleteStore)(JNIEnv* env, jobject self, jlong plan, jlong store, jintArray bucketIds,
                                             jlong literalsAddr, jint nLiterals) {
  (void)self;
  jint* ids = NULL;
  jsize n = 0;
  if (bucketIds != NULL) {
    n = (*env)->GetArrayLength(env, bucketIds);
    ids = (*env)->GetIntArrayElements(env, bucketIds, NULL);
    if (ids == NULL) return 0;                               /* OutOfMemoryError is pending */
  }
  int64_t rows = 0;
  int rc = sd_plan_delete_store((sd_plan*)(intptr_t)plan, (sd_store*)(intptr_t)store, (const int32_t*)ids, (int32_t)n,
                                (const sd_literal*)(intptr_t)literalsAddr, nLiterals, &rows);
  if (ids) (*env)->ReleaseIntArrayElements(env, bucketIds, ids, JNI_ABORT);
  if (rc) throw_last(env);
  return (jlong)rows;
}

/* compaction: folds update deltas and delete masks back into the base columns (sd_store_compact); out (length >= 4):
 * batches rewritten, batches removed, deleted rows purged, bytes written to the store's arena */
JNIEXPORT void JNICALL JFN(compactStore)(JNIEnv* env, jobject self, jlong store, jintArray bucketIds, jdouble minDirtyFraction,
                                         jlongArray out) {
  (void)self;
  if (out == NULL || (*env)->GetArrayLength(env, out) < 4) {
    throw_msg(env, "java/lang/IllegalArgumentException", "compactStore: out must hold 4 longs");
    return;
  }
  jint* ids = NULL;
  jsize n = 0;
  if (bucketIds != NULL) {
    n = (*env)->GetArrayLength(env, bucketIds);
    ids = (*env)->GetIntArrayElements(env, bucketIds, NULL);
    if (ids == NULL) return;                                  /* OutOfMemoryError is pending */
  }
  int64_t counts[4] = {0, 0, 0, 0};
  int rc = sd_store_compact((sd_store*)(intptr_t)store, (const int32_t*)ids, (int32_t)n, (double)minDirtyFraction, counts);
  if (ids) (*env)->ReleaseIntArrayElements(env, bucketIds, ids, JNI_ABORT);
  if (rc) { throw_last(env); return; }
  jlong o[4] = {(jlong)counts[0], (jlong)counts[1], (jlong)counts[2], (jlong)counts[3]};
  (*env)->SetLongArrayRegion(env, out, 0, 4, o);
}

/* reclaim: frees the device memory of superseded batch versions, after a compaction typically (sd_store_reclaim); out
 * (length >= 4): slabs freed, slab bytes freed, bytes copied, slabs deferred (an unfinished scan still reads them) */
JNIEXPORT void JNICALL JFN(reclaimStore)(JNIEnv* env, jobject self, jlong store, jdouble maxLiveFraction, jlongArray out) {
  (void)self;
  if (out == NULL || (*env)->GetArrayLength(env, out) < 4) {
    throw_msg(env, "java/lang/IllegalArgumentException", "reclaimStore: out must hold 4 longs");
    return;
  }
  int64_t counts[4] = {0, 0, 0, 0};
  if (sd_store_reclaim((sd_store*)(intptr_t)store, (double)maxLiveFraction, counts)) { throw_last(env); return; }
  jlong o[4] = {(jlong)counts[0], (jlong)counts[1], (jlong)counts[2], (jlong)counts[3]};
  (*env)->SetLongArrayRegion(env, out, 0, 4, o);
}

/* ---- the cross-partition exchange (INTEGRATION.md section 4b) ------------------------------------------------------ */
/* rank 0 fills a 128-byte id; the caller broadcasts it (a Spark broadcast variable) */
JNIEXPORT void JNICALL JFN(commUniqueId)(JNIEnv* env, jobject self, jbyteArray out128) {
  (void)self;
  uint8_t id[128];
  if (out128 == NULL || (*env)->GetArrayLength(env, out128) < 128) { throw_msg(env, "java/lang/IllegalArgumentException", "commUniqueId: byte[128]"); return; }
  if (sd_comm_unique_id(id)) { throw_last(env); return; }
  (*env)->SetByteArrayRegion(env, out128, 0, 128, (const jbyte*)id);
}
JNIEXPORT jlong JNICALL JFN(commCreate)(JNIEnv* env, jobject self, jbyteArray id128, jint rank, jint world, jint device) {
  (void)self;
  uint8_t id[128];
  sd_comm* c = NULL;
  if (id128 == NULL || (*env)->GetArrayLength(env, id128) < 128) { throw_msg(env, "java/lang/IllegalArgumentException", "commCreate: byte[128]"); return 0; }
  (*env)->GetByteArrayRegion(env, id128, 0, 128, (jbyte*)id);
  if ((*env)->ExceptionCheck(env)) return 0;
  if (sd_comm_create(id, rank, world, device, &c)) { throw_last(env); return 0; }   /* blocks until every rank has joined: no JNI state is held */
  return (jlong)(intptr_t)c;
}
JNIEXPORT void JNICALL JFN(commDestroy)(JNIEnv* env, jobject self, jlong comm) {
  (void)env; (void)self;
  sd_comm_destroy((sd_comm*)(intptr_t)comm);
}
/* all-gather + merge of this partition's partial result with the other ranks'; planFinish then returns the merged partial rows */
JNIEXPORT void JNICALL JFN(planExchange)(JNIEnv* env, jobject self, jlong plan, jlong comm) {
  (void)self;
  if (sd_plan_exchange((sd_plan*)(intptr_t)plan, (sd_comm*)(intptr_t)comm)) throw_last(env);
}

/* ---- page-locked host memory: result buffers of planFinish (projected rows arrive by ONE device->host copy at link speed) and
 *      long-lived staging.  The address is wrapped on the Scala side with Platform / a direct ByteBuffer view. ---------------- */
JNIEXPORT jlong JNICALL JFN(hostAlloc)(JNIEnv* env, jobject self, jlong bytes) {
  (void)self;
  void* p = NULL;
  if (sd_host_alloc(bytes, &p)) { throw_last(env); return 0; }
  return (jlong)(intptr_t)p;
}
JNIEXPORT void JNICALL JFN(hostFree)(JNIEnv* env, jobject self, jlong addr) {
  (void)env; (void)self;
  sd_host_free((void*)(intptr_t)addr);
}

JNIEXPORT void JNICALL JFN(rowsSubmit)(JNIEnv* env, jobject self, jlong plan, jlong rowsAddr, jlong len, jint nrows) {
  (void)self;
  if (sd_rows_submit((sd_plan*)(intptr_t)plan, (const void*)(intptr_t)rowsAddr, len, nrows)) throw_last(env);
}

/* returns the number of bytes written to outAddr; a negative value -needed when the buffer is too small */
JNIEXPORT jlong JNICALL JFN(planFinish)(JNIEnv* env, jobject self, jlong plan, jlong outAddr, jlong cap) {
  (void)self;
  int64_t len = 0, nrows = 0;
  int rc = sd_plan_finish((sd_plan*)(intptr_t)plan, (void*)(intptr_t)outAddr, cap, &len, &nrows);
  if (rc == SD_ERR_OVERFLOW) return -len;
  if (rc) { throw_last(env); return 0; }
  return len;
}

JNIEXPORT void JNICALL JFN(planReset)(JNIEnv* env, jobject self, jlong plan) {
  (void)self;
  if (sd_plan_reset((sd_plan*)(intptr_t)plan)) throw_last(env);
}

JNIEXPORT void JNICALL JFN(planMetrics)(JNIEnv* env, jobject self, jlong plan, jlongArray out) {
  (void)self;
  int64_t m[SD_NUM_METRICS];
  if (out == NULL || (*env)->GetArrayLength(env, out) < SD_NUM_METRICS) { throw_msg(env, "java/lang/IllegalArgumentException", "planMetrics: long[12]"); return; }
  if (sd_plan_metrics((sd_plan*)(intptr_t)plan, m)) { throw_last(env); return; }
  (*env)->SetLongArrayRegion(env, out, 0, SD_NUM_METRICS, (const jlong*)m);
}

JNIEXPORT void JNICALL JFN(planDestroy)(JNIEnv* env, jobject self, jlong plan) {
  (void)env; (void)self;
  sd_plan_destroy((sd_plan*)(intptr_t)plan);
}

JNIEXPORT jlong JNICALL JFN(finalMerge)(JNIEnv* env, jobject self, jlong planDescAddr, jlong rowsAddr, jlong len, jlong outAddr, jlong cap) {
  (void)self;
  int64_t olen = 0, nrows = 0;
  int rc = sd_final_merge((const sd_plan_desc*)(intptr_t)planDescAddr, (const void*)(intptr_t)rowsAddr, len,
                          (void*)(intptr_t)outAddr, cap, &olen, &nrows);
  if (rc == SD_ERR_OVERFLOW) return -olen;
  if (rc) { throw_last(env); return 0; }
  return olen;
}
