"""Host-side writer/reader of SnappyData's ColumnBatch byte format.

This is the *format specification* the rest of the engine is built against: it produces the exact
bytes the reference's column encoders put into a ``ColumnFormatValue`` so that the CUDA path, the
CPU oracle and the tests all consume identical ColumnBatch bytes.  It is a restatement written from
the layouts, not a translation of the encoder classes; citations are to /root/reference:

  enc = encoders/src/main/scala/org/apache/spark/sql/execution/columnar/encoding

  column buffer   [typeId:int32][nullBytes:int32][null words:int64 x W][body]     enc/ColumnEncoding.scala:37-54
                  null words are trimmed of trailing zero words                    enc/ColumnEncoding.scala:1192-1196,1267-1322
                  body holds NON-NULL values only                                  enc/ColumnEncoding.scala:1103-1142
  Uncompressed    packed little-endian fixed-width values                          enc/Uncompressed.scala:74-98
  Dictionary      [numElements:int32][dictionary][int16|int32 index per non-null]  enc/DictionaryEncoding.scala:85-166,351-430
                  switch to int32 indexes (typeId 3) when index 32767 is reached   enc/DictionaryEncoding.scala:313-318
  BooleanBitSet   int64 words, bit k = k-th non-null value                         enc/BooleanBitSetEncoding.scala:57-59
  RunLength       [value][runLength:int32] runs (decoder-defined only)             enc/RunLengthEncoding.scala:99-172
  update delta    header+nulls, [numBaseRows][numDeltas][positions], pad 8, values enc/ColumnDeltaEncoder.scala:300-331
  delete mask     [0][numBaseRows][numDeletes][positions]                          enc/ColumnDeleteEncoder.scala:101-134
  stats row       Spark UnsafeRow [batchCount,(lower,upper,nullCount) x ncols]     enc/ColumnEncoding.scala:1015-1036
  compression     [-codecId][uncompressedLen][payload]                             encoders/.../store/CompressionUtils.scala:53-61

All multi-byte values are little-endian.
"""
from __future__ import annotations

import ctypes
import ctypes.util
import enum
import struct
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

# ---- encoding type ids (enc/ColumnEncoding.scala:766-773) -------------------------------------
UNCOMPRESSED = 0
RUN_LENGTH = 1
DICTIONARY = 2
BIG_DICTIONARY = 3
BOOLEAN_BITSET = 4

# column index keys of the auxiliary buffers of a batch (encoders/.../impl/ColumnFormatEntry.scala:79-87)
STATROW_COL_INDEX = -1
DELTA_STATROW_COL_INDEX = -2
DELETE_MASK_COL_INDEX = -3

MAX_ROWS_IN_BATCH = 200000  # jdbc/src/main/scala/io/snappydata/Constant.scala:142


class SqlType(enum.IntEnum):
    """SQL types of scan columns; values match ``sd_type_t`` in include/snappy_gpu.h."""
    BOOLEAN = 1
    BYTE = 2
    SHORT = 3
    INT = 4
    LONG = 5
    FLOAT = 6
    DOUBLE = 7
    DATE = 8        # int32 days since epoch
    TIMESTAMP = 9   # int64 microseconds since epoch
    STRING = 10
    DECIMAL = 11    # precision <= 18: int64 unscaled value


_NP_DTYPE = {
    SqlType.BOOLEAN: np.dtype("u1"), SqlType.BYTE: np.dtype("i1"), SqlType.SHORT: np.dtype("<i2"),
    SqlType.INT: np.dtype("<i4"), SqlType.LONG: np.dtype("<i8"), SqlType.FLOAT: np.dtype("<f4"),
    SqlType.DOUBLE: np.dtype("<f8"), SqlType.DATE: np.dtype("<i4"), SqlType.TIMESTAMP: np.dtype("<i8"),
    SqlType.DECIMAL: np.dtype("<i8"),
}


def np_dtype(t: SqlType) -> np.dtype:
    return _NP_DTYPE[SqlType(t)]


def fixed_width(t: SqlType) -> int:
    return _NP_DTYPE[SqlType(t)].itemsize


# ---- null bitmap -----------------------------------------------------------------------------
def null_words(nulls: Optional[np.ndarray]) -> np.ndarray:
    """LE 64-bit words, bit (i & 63) of word (i >> 6) set <=> row i is NULL; trailing zero words
    trimmed (enc/ColumnEncoding.scala:1192-1196)."""
    if nulls is None:
        return np.zeros(0, dtype="<u8")
    nulls = np.asarray(nulls, dtype=bool)
    if not nulls.any():
        return np.zeros(0, dtype="<u8")
    n = nulls.shape[0]
    padded = np.zeros(((n + 63) // 64) * 64, dtype=np.uint8)
    padded[:n] = nulls
    words = np.packbits(padded.reshape(-1, 8), axis=1, bitorder="little").reshape(-1, 8)
    words = np.ascontiguousarray(words).view("<u8").reshape(-1)
    nz = np.nonzero(words)[0]
    return words[: int(nz[-1]) + 1].copy()


def _header(type_id: int, nwords: np.ndarray) -> bytes:
    return struct.pack("<ii", type_id, 8 * len(nwords)) + nwords.tobytes()


def _non_null(values: np.ndarray, nulls: Optional[np.ndarray]) -> np.ndarray:
    if nulls is None:
        return values
    nulls = np.asarray(nulls, dtype=bool)
    return values[~nulls]


# ---- encoders --------------------------------------------------------------------------------
def encode_uncompressed(values, sql_type: SqlType, nulls=None) -> bytes:
    """typeId 0; fixed-width types and (for STRING) back-to-back [int32 len][bytes]."""
    sql_type = SqlType(sql_type)
    nw = null_words(nulls)
    if sql_type == SqlType.STRING:
        vals = [v for i, v in enumerate(values) if nulls is None or not nulls[i]]
        body = b"".join(struct.pack("<i", len(_b(v))) + _b(v) for v in vals)
        return _header(UNCOMPRESSED, nw) + body
    arr = np.asarray(values)
    if sql_type == SqlType.BOOLEAN:
        arr = arr.astype(bool).astype("u1")
    arr = _non_null(arr, nulls).astype(np_dtype(sql_type), copy=False)
    return _header(UNCOMPRESSED, nw) + arr.tobytes()


def decimal_bytes(unscaled: int) -> bytes:
    """BigInteger.toByteArray(): the minimal big-endian two's complement of an unscaled DECIMAL value."""
    n = (int(unscaled) + (unscaled < 0)).bit_length() // 8 + 1
    return int(unscaled).to_bytes(n, "big", signed=True)


def encode_wide_decimal(values, nulls=None) -> bytes:
    """typeId 0 for DECIMAL(p > 18): back-to-back [int32 len][BigInteger bytes] of the non-null unscaled values
    (enc/Uncompressed.scala:330-345)."""
    nw = null_words(nulls)
    vals = [int(v) for i, v in enumerate(values) if nulls is None or not nulls[i]]
    return _header(UNCOMPRESSED, nw) + b"".join(struct.pack("<i", len(decimal_bytes(v))) + decimal_bytes(v) for v in vals)


def wide_decimal_stats(values, precision: int, scale: int, nulls=None):
    """column_stats for DECIMAL(p > 18): bounds are unscaled ints, typed (DECIMAL, precision, scale) for the stats row."""
    vals = [int(v) for i, v in enumerate(values) if nulls is None or not nulls[i]]
    nc = int(np.count_nonzero(nulls)) if nulls is not None else 0
    t = (SqlType.DECIMAL, precision, scale)
    return (t, min(vals), max(vals), nc) if vals else (t, None, None, nc)


def _b(v) -> bytes:
    return v if isinstance(v, (bytes, bytearray, np.bytes_)) else str(v).encode("utf-8")


def _first_seen_dictionary(arr: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """Distinct values of ``arr`` in first-seen order plus the per-element index (the reference's
    DictionaryMap / ObjectHashSet hands out indexes in insertion order,
    enc/DictionaryEncoding.scala:296-349)."""
    if arr.shape[0] == 0:
        return arr[:0], np.zeros(0, dtype=np.int64)
    uniq, first, inv = np.unique(arr, return_index=True, return_inverse=True)
    order = np.argsort(first, kind="stable")          # unique ids ordered by first occurrence
    rank = np.empty_like(order)
    rank[order] = np.arange(order.shape[0])
    return uniq[order], rank[inv.reshape(-1)]


def encode_dictionary(values, sql_type: SqlType, nulls=None, force_big: bool = False) -> bytes:
    """typeId 2 (int16 indexes) or 3 (int32 indexes) for STRING / INT / DATE / LONG / TIMESTAMP."""
    sql_type = SqlType(sql_type)
    nw = null_words(nulls)
    if sql_type == SqlType.STRING:
        arr = np.asarray([_b(v) for v in values], dtype=object) if not (
            isinstance(values, np.ndarray) and values.dtype.kind == "S") else values
        arr = _non_null(np.asarray(arr), nulls)
        if arr.dtype.kind != "S":
            maxlen = max((len(x) for x in arr), default=1)
            # np 'S' strips trailing NULs; dictionary strings containing them are not supported here
            arr = arr.astype(f"S{max(maxlen, 1)}")
        dict_vals, idx = _first_seen_dictionary(arr)
        dict_bytes = b"".join(struct.pack("<i", len(bytes(s))) + bytes(s) for s in dict_vals)
    elif sql_type in (SqlType.INT, SqlType.DATE):
        arr = _non_null(np.asarray(values), nulls).astype("<i4")
        dict_vals, idx = _first_seen_dictionary(arr)
        dict_bytes = dict_vals.astype("<i4").tobytes()
    elif sql_type in (SqlType.LONG, SqlType.TIMESTAMP):
        arr = _non_null(np.asarray(values), nulls).astype("<i8")
        dict_vals, idx = _first_seen_dictionary(arr)
        # written 8 bytes/entry (allocation slack of the reference is at the buffer tail and
        # does not affect decode, enc/DictionaryEncoding.scala:374-379,393-394)
        dict_bytes = dict_vals.astype("<i8").tobytes()
    else:
        raise ValueError(f"dictionary encoding not supported for {sql_type!r}")
    n = int(dict_vals.shape[0])
    # index Short.MaxValue (32767) triggers the switch to the big dictionary
    big = force_big or n > 32767
    body = struct.pack("<i", n) + dict_bytes + idx.astype("<i4" if big else "<i2").tobytes()
    return _header(BIG_DICTIONARY if big else DICTIONARY, nw) + body


def encode_boolean_bitset(values, nulls=None) -> bytes:
    """typeId 4: bit k of the LE 64-bit words = k-th non-null value."""
    nw = null_words(nulls)
    arr = _non_null(np.asarray(values).astype(bool), nulls)
    n = arr.shape[0]
    padded = np.zeros(((n + 63) // 64) * 64, dtype=np.uint8)
    padded[:n] = arr
    words = np.packbits(padded.reshape(-1, 8), axis=1, bitorder="little")
    return _header(BOOLEAN_BITSET, nw) + np.ascontiguousarray(words).tobytes()


def encode_run_length(values, sql_type: SqlType, nulls=None) -> bytes:
    """typeId 1 as *defined by the decoder* (no encoder exists in the reference):
    runs of [value][runLength:int32]; SHORT 2+4, INT/DATE 4+4, LONG/TIMESTAMP 8+4,
    STRING [len][bytes][run]  (enc/RunLengthEncoding.scala:112-172).
    BYTE/BOOLEAN are refused: the reference decoder advances 3 bytes after a 1+4 byte run
    (enc/RunLengthEncoding.scala:99-110), so no byte layout decodes consistently."""
    sql_type = SqlType(sql_type)
    nw = null_words(nulls)
    if sql_type == SqlType.STRING:
        vals = [_b(v) for i, v in enumerate(values) if nulls is None or not nulls[i]]
        out = bytearray()
        i = 0
        while i < len(vals):
            j = i
            while j + 1 < len(vals) and vals[j + 1] == vals[i]:
                j += 1
            out += struct.pack("<i", len(vals[i])) + vals[i] + struct.pack("<i", j - i + 1)
            i = j + 1
        return _header(RUN_LENGTH, nw) + bytes(out)
    if sql_type in (SqlType.BYTE, SqlType.BOOLEAN):
        raise ValueError("RunLength BYTE/BOOLEAN: reference decoder is inconsistent; refused")
    if sql_type not in (SqlType.SHORT, SqlType.INT, SqlType.DATE, SqlType.LONG, SqlType.TIMESTAMP):
        raise ValueError(f"run-length encoding not supported for {sql_type!r}")
    arr = _non_null(np.asarray(values), nulls).astype(np_dtype(sql_type))
    if arr.shape[0] == 0:
        return _header(RUN_LENGTH, nw)
    change = np.flatnonzero(np.concatenate(([True], arr[1:] != arr[:-1])))
    lengths = np.diff(np.concatenate((change, [arr.shape[0]]))).astype("<i4")
    w = arr.dtype.itemsize
    rec = np.zeros((change.shape[0], w + 4), dtype=np.uint8)
    rec[:, :w] = arr[change].view(np.uint8).reshape(-1, w)
    rec[:, w:] = lengths.view(np.uint8).reshape(-1, 4)
    return _header(RUN_LENGTH, nw) + rec.tobytes()


def encode_column(values, sql_type: SqlType, nulls=None) -> bytes:
    """Default encoder choice of the reference (enc/ColumnEncoding.scala:837-844):
    STRING -> Dictionary, BOOLEAN -> BooleanBitSet, everything else Uncompressed."""
    sql_type = SqlType(sql_type)
    if sql_type == SqlType.STRING:
        return encode_dictionary(values, sql_type, nulls)
    if sql_type == SqlType.BOOLEAN:
        return encode_boolean_bitset(values, nulls)
    return encode_uncompressed(values, sql_type, nulls)


def encode_delta(num_base_rows: int, positions, values, sql_type: SqlType, nulls=None,
                 dictionary: Optional[bool] = None) -> bytes:
    """Update-delta buffer: normal header whose null bits index the *relative* delta entry, then
    [numBaseRows][numDeltas][positions asc], pad to 8, then the values in the column's normal
    encoding (enc/ColumnDeltaEncoder.scala:300-331, enc/ColumnDeltaDecoder.scala:47-61)."""
    positions = np.asarray(positions, dtype="<i4")
    assert np.all(np.diff(positions) > 0), "delta positions must be strictly ascending"
    sql_type = SqlType(sql_type)
    if dictionary is None:
        dictionary = sql_type == SqlType.STRING
    if dictionary:
        enc = encode_dictionary(values, sql_type, nulls)
    elif sql_type == SqlType.BOOLEAN:
        enc = encode_boolean_bitset(values, nulls)
    else:
        enc = encode_uncompressed(values, sql_type, nulls)
    type_id, null_bytes = struct.unpack_from("<ii", enc, 0)
    head = enc[: 8 + null_bytes]
    body = enc[8 + null_bytes:]
    mid = struct.pack("<ii", num_base_rows, positions.shape[0]) + positions.tobytes()
    pad = (-(len(head) + len(mid))) % 8
    return head + mid + b"\0" * pad + body


def encode_delete(num_base_rows: int, positions) -> bytes:
    """Delete mask: [reserved=0][numBaseRows][numDeletes][positions asc]
    (enc/ColumnDeleteEncoder.scala:101-134)."""
    positions = np.asarray(positions, dtype="<i4")
    assert np.all(np.diff(positions) > 0), "delete positions must be strictly ascending"
    return struct.pack("<iii", 0, num_base_rows, positions.shape[0]) + positions.tobytes()


# ---- Spark UnsafeRow (Appendix B.9 of SURVEY.md) -----------------------------------------------
def unsafe_row(fields: Sequence[Tuple[SqlType, object]]) -> bytes:
    """ceil(n/64)*8 bytes of null bits, n 8-byte slots, then 8-byte padded variable-length data;
    a var-length slot holds (offsetFromRowBase << 32) | sizeInBytes."""
    n = len(fields)
    bitset = bytearray(((n + 63) // 64) * 8)
    slots = bytearray(8 * n)
    var = bytearray()
    fixed_len = len(bitset) + len(slots)
    for i, (t, v) in enumerate(fields):
        wide = isinstance(t, tuple) and t[1] > 18   # (DECIMAL, precision, scale): BigInteger bytes in a 16-byte region
        t = SqlType(t[0] if isinstance(t, tuple) else t)
        if v is None:
            bitset[i >> 3] |= 1 << (i & 7)
            continue
        off = 8 * i
        if wide:
            b = decimal_bytes(v)
            struct.pack_into("<q", slots, off, ((fixed_len + len(var)) << 32) | len(b))
            var += b + b"\0" * (16 - len(b))
        elif t == SqlType.STRING:
            b = _b(v)
            struct.pack_into("<q", slots, off, ((fixed_len + len(var)) << 32) | len(b))
            var += b + b"\0" * ((-len(b)) % 8)
        elif t == SqlType.BOOLEAN:
            slots[off] = 1 if v else 0
        elif t == SqlType.BYTE:
            struct.pack_into("<b", slots, off, int(v))
        elif t == SqlType.SHORT:
            struct.pack_into("<h", slots, off, int(v))
        elif t in (SqlType.INT, SqlType.DATE):
            struct.pack_into("<i", slots, off, int(v))
        elif t in (SqlType.LONG, SqlType.TIMESTAMP, SqlType.DECIMAL):
            struct.pack_into("<q", slots, off, int(v))
        elif t == SqlType.FLOAT:
            struct.pack_into("<f", slots, off, float(v))
        elif t == SqlType.DOUBLE:
            struct.pack_into("<d", slots, off, float(v))
        else:
            raise ValueError(t)
    return bytes(bitset) + bytes(slots) + bytes(var)


def parse_unsafe_row(buf: bytes, types: Sequence[object], base: int = 0) -> List[object]:
    """`types`: SqlType per field, or (SqlType.DECIMAL, precision, scale) -- a DECIMAL comes back as its unscaled int
    (precision > 18: BigInteger bytes in the variable-length region, UnsafeRow.getDecimal)."""
    n = len(types)
    bitset_len = ((n + 63) // 64) * 8
    out: List[object] = []
    for i, t in enumerate(types):
        prec = 18
        if isinstance(t, tuple):
            t, prec = t[0], t[1]
        t = SqlType(t)
        if buf[base + (i >> 3)] & (1 << (i & 7)):
            out.append(None)
            continue
        off = base + bitset_len + 8 * i
        if t == SqlType.DECIMAL and prec > 18:
            (ol,) = struct.unpack_from("<q", buf, off)
            o, ln = ol >> 32, ol & 0xFFFFFFFF
            out.append(int.from_bytes(bytes(buf[base + o: base + o + ln]), "big", signed=True))
        elif t == SqlType.STRING:
            (ol,) = struct.unpack_from("<q", buf, off)
            o, ln = ol >> 32, ol & 0xFFFFFFFF
            out.append(bytes(buf[base + o: base + o + ln]))
        elif t == SqlType.BOOLEAN:
            out.append(buf[off] != 0)
        elif t == SqlType.BYTE:
            out.append(struct.unpack_from("<b", buf, off)[0])
        elif t == SqlType.SHORT:
            out.append(struct.unpack_from("<h", buf, off)[0])
        elif t in (SqlType.INT, SqlType.DATE):
            out.append(struct.unpack_from("<i", buf, off)[0])
        elif t in (SqlType.LONG, SqlType.TIMESTAMP, SqlType.DECIMAL):
            out.append(struct.unpack_from("<q", buf, off)[0])
        elif t == SqlType.FLOAT:
            out.append(struct.unpack_from("<f", buf, off)[0])
        elif t == SqlType.DOUBLE:
            out.append(struct.unpack_from("<d", buf, off)[0])
        else:
            raise ValueError(t)
    return out


def parse_row_stream(buf: bytes, types: Sequence[SqlType]) -> List[List[object]]:
    """Rows as emitted by ``sd_plan_finish``: repeated [int64 sizeInBytes][UnsafeRow bytes]."""
    rows, pos = [], 0
    while pos < len(buf):
        (sz,) = struct.unpack_from("<q", buf, pos)
        rows.append(parse_unsafe_row(buf, types, pos + 8))
        pos += 8 + sz
    return rows


def stats_row(batch_count: int, col_stats: Sequence[Tuple[SqlType, object, object, int]],
              has_deltas: bool = False) -> bytes:
    """Stats UnsafeRow: [batchCount:int (negative => batch has update deltas),
    (lowerBound, upperBound, nullCount:int) per table column]
    (enc/ColumnEncoding.scala:1015-1036; core/.../ColumnTableScan.scala:518-531)."""
    fields: List[Tuple[SqlType, object]] = [(SqlType.INT, -batch_count if has_deltas else batch_count)]
    for t, lo, hi, nc in col_stats:
        fields += [(t, lo), (t, hi), (SqlType.INT, int(nc))]
    return unsafe_row(fields)


def column_stats(values, sql_type: SqlType, nulls=None) -> Tuple[SqlType, object, object, int]:
    """(type, lower, upper, nullCount) as ColumnWriter records them
    (core/.../ColumnInsertExec.scala:848-921); bounds are None for an all-null column."""
    sql_type = SqlType(sql_type)
    nc = int(np.count_nonzero(nulls)) if nulls is not None else 0
    if sql_type == SqlType.STRING:
        vals = [_b(v) for i, v in enumerate(values) if nulls is None or not nulls[i]]
        if not vals:
            return (sql_type, None, None, nc)
        return (sql_type, min(vals), max(vals), nc)
    arr = _non_null(np.asarray(values), nulls)
    if arr.shape[0] == 0:
        return (sql_type, None, None, nc)
    if sql_type == SqlType.BOOLEAN:
        return (sql_type, bool(arr.min()), bool(arr.max()), nc)
    lo, hi = arr.min(), arr.max()
    if sql_type in (SqlType.FLOAT, SqlType.DOUBLE):
        return (sql_type, float(lo), float(hi), nc)
    return (sql_type, int(lo), int(hi), nc)


# ---- compression envelope (encoders/.../store/CompressionUtils.scala:53-61,102-110) -----------
CODEC_LZ4 = 1
CODEC_SNAPPY = 2
COMPRESSION_MIN_SIZE = 2048

_lz4 = None


def _liblz4():
    global _lz4
    if _lz4 is None:
        name = ctypes.util.find_library("lz4") or "liblz4.so.1"
        lib = ctypes.CDLL(name)
        lib.LZ4_compress_default.restype = ctypes.c_int
        lib.LZ4_compress_default.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.c_int, ctypes.c_int]
        lib.LZ4_decompress_safe.restype = ctypes.c_int
        lib.LZ4_decompress_safe.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.c_int, ctypes.c_int]
        lib.LZ4_compressBound.restype = ctypes.c_int
        lib.LZ4_compressBound.argtypes = [ctypes.c_int]
        _lz4 = lib
    return _lz4


def compress_lz4(buf: bytes, force: bool = False) -> bytes:
    """[-1][uncompressedLen][LZ4 block]; stored compressed only if >= 2048 B and the result is
    <= 75 % of the input (CompressionUtils.scala:47-49,102-110) unless ``force``."""
    if len(buf) < COMPRESSION_MIN_SIZE and not force:
        return buf
    lib = _liblz4()
    cap = lib.LZ4_compressBound(len(buf))
    dst = ctypes.create_string_buffer(cap)
    n = lib.LZ4_compress_default(buf, dst, len(buf), cap)
    if n <= 0 or (not force and n > (len(buf) * 3) // 4):
        return buf
    return struct.pack("<ii", -CODEC_LZ4, len(buf)) + dst.raw[:n]


def compress_snappy(buf: bytes) -> bytes:
    """[-2][uncompressedLen][Snappy raw stream] (CompressionCodecId.SNAPPY_ID = 2, CompressionUtils.scala:125-168).
    A small greedy encoder for fixtures (no snappy library in this image): varint length, then literals and 2-byte-offset
    copies found through a hash of 4-byte windows -- every element kind the decoder must handle except 4-byte offsets."""
    n = len(buf)
    out = bytearray()
    v = n
    while True:
        b = v & 0x7F
        v >>= 7
        out.append(b | (0x80 if v else 0))
        if not v:
            break

    def literal(lo, hi):
        while lo < hi:
            ln = min(hi - lo, 1 << 16)
            if ln <= 60:
                out.append((ln - 1) << 2)
            elif ln <= 256:
                out.extend(bytes([60 << 2, ln - 1]))
            else:
                out.extend(bytes([61 << 2, (ln - 1) & 0xFF, (ln - 1) >> 8]))
            out.extend(buf[lo:lo + ln])
            lo += ln

    table = {}
    i = lit = 0
    while i + 4 <= n:
        key = buf[i:i + 4]
        j = table.get(key)
        table[key] = i
        if j is not None and 0 < i - j < 65536:
            ln = 4
            while i + ln < n and ln < 64 and buf[j + ln] == buf[i + ln]:
                ln += 1
            literal(lit, i)
            off = i - j
            if 4 <= ln <= 11 and off < 2048:
                out += bytes([1 | ((ln - 4) << 2) | ((off >> 8) << 5), off & 0xFF])
            else:
                out += bytes([2 | ((ln - 1) << 2), off & 0xFF, off >> 8])
            i += ln
            lit = i
        else:
            i += 1
    literal(lit, n)
    return struct.pack("<ii", -CODEC_SNAPPY, n) + bytes(out)


def decompress(buf: bytes) -> bytes:
    (first,) = struct.unpack_from("<i", buf, 0)
    if first >= 0:
        return buf
    if -first != CODEC_LZ4:
        raise ValueError(f"codec {-first} not available in this environment")
    (ulen,) = struct.unpack_from("<i", buf, 4)
    dst = ctypes.create_string_buffer(ulen)
    n = _liblz4().LZ4_decompress_safe(bytes(buf[8:]), dst, len(buf) - 8, ulen)
    if n != ulen:
        raise ValueError("corrupt LZ4 payload")
    return dst.raw


# ---- numpy decoders (host-side reader, used by tests and the Python oracle) -------------------
def parse_header(buf: bytes) -> Tuple[int, np.ndarray, int]:
    """-> (typeId, null words, body offset)."""
    type_id, null_bytes = struct.unpack_from("<ii", buf, 0)
    assert null_bytes % 8 == 0
    words = np.frombuffer(buf, dtype="<u8", count=null_bytes // 8, offset=8)
    return type_id, words, 8 + null_bytes


def nulls_from_words(words: np.ndarray, num_rows: int) -> np.ndarray:
    out = np.zeros(num_rows, dtype=bool)
    if words.shape[0]:
        bits = np.unpackbits(words.view(np.uint8), bitorder="little").astype(bool)
        m = min(num_rows, bits.shape[0])
        out[:m] = bits[:m]
    return out


def decode_column(buf: bytes, sql_type: SqlType, num_rows: int, _delta_skip: int = 0):
    """Decode a column buffer -> (values, nulls).  Values at NULL rows are 0 / b''.
    STRING columns decode to an object array of ``bytes``."""
    sql_type = SqlType(sql_type)
    buf = decompress(bytes(buf))
    type_id, words, pos = parse_header(buf)
    pos += _delta_skip
    nulls = nulls_from_words(words, num_rows)
    nn = int(num_rows - nulls.sum())
    if type_id == UNCOMPRESSED:
        if sql_type == SqlType.STRING:
            vals = []
            for _ in range(nn):
                (ln,) = struct.unpack_from("<i", buf, pos)
                vals.append(bytes(buf[pos + 4: pos + 4 + ln]))
                pos += 4 + ln
            dense = np.asarray(vals + [b""], dtype=object)[:-1]
        else:
            dense = np.frombuffer(buf, dtype=np_dtype(sql_type), count=nn, offset=pos)
            if sql_type == SqlType.BOOLEAN:
                dense = dense == 1
    elif type_id in (DICTIONARY, BIG_DICTIONARY):
        (n,) = struct.unpack_from("<i", buf, pos)
        pos += 4
        if sql_type == SqlType.STRING:
            d = []
            for _ in range(n):
                (ln,) = struct.unpack_from("<i", buf, pos)
                d.append(bytes(buf[pos + 4: pos + 4 + ln]))
                pos += 4 + ln
            dvals = np.asarray(d + [b""], dtype=object)[:-1]
        elif sql_type in (SqlType.INT, SqlType.DATE):
            dvals = np.frombuffer(buf, dtype="<i4", count=n, offset=pos)
            pos += 4 * n
        else:
            dvals = np.frombuffer(buf, dtype="<i8", count=n, offset=pos)
            pos += 8 * n
        idx = np.frombuffer(buf, dtype="<i2" if type_id == DICTIONARY else "<i4", count=nn, offset=pos)
        dense = dvals[idx.astype(np.int64)] if nn else dvals[:0]
    elif type_id == BOOLEAN_BITSET:
        nw = (nn + 63) // 64
        w = np.frombuffer(buf, dtype="<u8", count=nw, offset=pos)
        dense = np.unpackbits(w.view(np.uint8), bitorder="little").astype(bool)[:nn]
    elif type_id == RUN_LENGTH:
        out = []
        if sql_type == SqlType.STRING:
            while len(out) < nn:
                (ln,) = struct.unpack_from("<i", buf, pos)
                v = bytes(buf[pos + 4: pos + 4 + ln])
                (run,) = struct.unpack_from("<i", buf, pos + 4 + ln)
                out += [v] * run
                pos += 8 + ln
            dense = np.asarray(out + [b""], dtype=object)[:-1]
        else:
            dt = np_dtype(sql_type)
            w = dt.itemsize
            vals, runs = [], []
            tot = 0
            while tot < nn:
                vals.append(np.frombuffer(buf, dtype=dt, count=1, offset=pos)[0])
                (run,) = struct.unpack_from("<i", buf, pos + w)
                runs.append(run)
                tot += run
                pos += w + 4
            dense = np.repeat(np.asarray(vals, dtype=dt), runs)[:nn] if vals else np.zeros(0, dt)
    else:
        raise ValueError(f"unknown encoding typeId {type_id}")
    if sql_type == SqlType.STRING:
        full = np.empty(num_rows, dtype=object)
        full[:] = b""
    elif sql_type == SqlType.BOOLEAN:
        full = np.zeros(num_rows, dtype=bool)
    else:
        full = np.zeros(num_rows, dtype=np_dtype(sql_type))
    full[~nulls] = dense
    return full, nulls


def decode_delta(buf: bytes, sql_type: SqlType):
    """-> (numBaseRows, positions, values, nulls) of an update-delta buffer."""
    buf = decompress(bytes(buf))
    _, words, pos = parse_header(buf)
    nbase, n = struct.unpack_from("<ii", buf, pos)
    positions = np.frombuffer(buf, dtype="<i4", count=n, offset=pos + 8).copy()
    end = pos + 8 + 4 * n
    data = ((end + 7) >> 3) << 3
    vals, nulls = decode_column(buf, sql_type, n, _delta_skip=data - pos)
    return nbase, positions, vals, nulls


def decode_delete(buf: bytes):
    buf = bytes(buf)
    _, nbase, n = struct.unpack_from("<iii", buf, 0)
    # the reference's decoder walks to the end of the buffer (enc/ColumnDeleteDecoder.scala:31-36)
    cnt = (len(buf) - 12) // 4
    return nbase, np.frombuffer(buf, dtype="<i4", count=cnt, offset=12).copy()


# ---- batch container ---------------------------------------------------------------------------
@dataclass
class ColumnBatch:
    """One column batch as the scan sees it (encoders/.../columnar/ColumnBatch.scala:36-50 plus the
    delta/delete buffers ColumnBatchIterator serves, core/.../ColumnBatchIterator.scala:122-163).
    ``columns`` is indexed by 0-based *table* column; entries may be None for columns never read."""
    num_rows: int
    columns: List[Optional[bytes]]
    stats: Optional[bytes] = None
    delta0: Dict[int, bytes] = field(default_factory=dict)   # table column -> depth-0 delta
    delta1: Dict[int, bytes] = field(default_factory=dict)   # table column -> depth-1 delta
    delete_mask: Optional[bytes] = None
    batch_id: int = 0
    bucket_id: int = 0

    @property
    def has_deltas(self) -> bool:
        return bool(self.delta0) or bool(self.delta1)

    def body_bytes(self, table_cols: Sequence[int]) -> int:
        """Algorithmic bytes of the referenced columns: buffer length - 8-byte header - dictionary
        bytes (SURVEY.md 8d)."""
        total = 0
        for c in table_cols:
            buf = self.columns[c]
            type_id, null_bytes = struct.unpack_from("<ii", buf, 0)
            n = len(buf) - 8
            if type_id in (DICTIONARY, BIG_DICTIONARY):
                n -= _dictionary_section_len(buf, 8 + null_bytes)
            total += n
        return total


def _dictionary_section_len(buf: bytes, pos: int) -> int:
    """Length of [numElements][dictionary] for a STRING dictionary; callers with int/long
    dictionaries must account for them separately (only used for accounting)."""
    (n,) = struct.unpack_from("<i", buf, pos)
    p = pos + 4
    for _ in range(n):
        (ln,) = struct.unpack_from("<i", buf, p)
        p += 4 + ln
    return p - pos


def build_batch(num_rows: int, schema: Sequence[Tuple[str, SqlType, bool]], data: Dict[str, object],
                nulls: Optional[Dict[str, np.ndarray]] = None, batch_id: int = 0, bucket_id: int = 0,
                encoders: Optional[Dict[str, str]] = None) -> ColumnBatch:
    """Encode one batch with the reference's default encoders (or per-column overrides:
    'uncompressed' | 'dictionary' | 'bigdictionary' | 'bitset' | 'rle') and build its stats row."""
    nulls = nulls or {}
    encoders = encoders or {}
    cols: List[Optional[bytes]] = []
    stats = []
    for name, t, nullable in schema:
        v = data[name]
        nl = nulls.get(name) if nullable else None
        enc = encoders.get(name)
        if enc is None:
            buf = encode_column(v, t, nl)
        elif enc == "uncompressed":
            buf = encode_uncompressed(v, t, nl)
        elif enc == "dictionary":
            buf = encode_dictionary(v, t, nl)
        elif enc == "bigdictionary":
            buf = encode_dictionary(v, t, nl, force_big=True)
        elif enc == "bitset":
            buf = encode_boolean_bitset(v, nl)
        elif enc == "rle":
            buf = encode_run_length(v, t, nl)
        else:
            raise ValueError(enc)
        cols.append(buf)
        stats.append(column_stats(v, t, nl))
    return ColumnBatch(num_rows=num_rows, columns=cols, stats=stats_row(num_rows, stats),
                       batch_id=batch_id, bucket_id=bucket_id)
