"""Split-image construction from documents (small, test-sized) and from the synthetic corpus spec.

This is NOT part of the search hot path. It stands where Quickwit's indexing pipeline + tantivy's
segment writer stand (out of scope, SURVEY.md §2): it turns documents into the postings /
fieldnorms / columns that `qwgpu_split_register` uploads. All byte-level encoding is done by the
C++ writer behind `qwgpu_imgb_*`; this module only tokenizes and groups.

Doc-mapping dialect: the subset of Quickwit's doc mapper JSON this path needs
(quickwit-doc-mapper/src/doc_mapper/field_mapping_entry.rs): `field_mappings[]` entries with
`name`, `type` (text|u64|i64|f64|bool|datetime|bytes), `tokenizer` (default|raw), `record`
(basic|freq|position; default basic, :447), `fieldnorms` (default false, :326), `fast`,
`fast_precision` (seconds|milliseconds|microseconds|nanoseconds), `input_format` (bytes: base64|hex,
default base64), plus `timestamp_field` and `mode: dynamic` (unknown JSON keys become fast raw-text /
numeric columns and raw-indexed text). A fast bytes field becomes a QW_COL_BYTES column: ordinals into
the sorted dictionary of its raw values.
"""
from __future__ import annotations

import base64
import ctypes as C
import datetime as _dt
import struct
from typing import Any, Dict, Iterable, List, Optional, Sequence

import numpy as np

from . import ffi

_PRECISION_NS = {"seconds": 10**9, "milliseconds": 10**6, "microseconds": 10**3, "nanoseconds": 1}


class SplitImage:
    """Owns the bytes of one split image (host memory)."""

    def __init__(self, buf: bytes | np.ndarray, split_id: str = ""):
        if isinstance(buf, np.ndarray):
            self.array = buf
        else:
            self.array = np.frombuffer(buf, dtype=np.uint8)
        self.split_id = split_id

    @property
    def ptr(self) -> int:
        return self.array.ctypes.data

    @property
    def nbytes(self) -> int:
        return int(self.array.nbytes)

    @property
    def num_docs(self) -> int:
        return self.header().num_docs

    def header(self) -> ffi.QwImgHeader:
        return ffi.QwImgHeader.from_buffer_copy(self.array[:C.sizeof(ffi.QwImgHeader)].tobytes())

    def _table(self, cls, off: int, n: int):
        sz = C.sizeof(cls)
        raw = self.array[off: off + sz * n].tobytes()
        return [cls.from_buffer_copy(raw[i * sz:(i + 1) * sz]) for i in range(n)]

    def _directory(self):
        if getattr(self, "_dir", None) is None:
            h = self.header()
            strings = self.array[h.strings_off: h.strings_off + h.strings_len].tobytes()
            tbytes = self.array[h.term_bytes_off: h.term_bytes_off + h.term_bytes_len].tobytes()
            fields = self._table(ffi.QwImgField, h.fields_off, h.num_fields)
            terms = self._table(ffi.QwImgTerm, h.terms_off, h.num_terms)
            cols = self._table(ffi.QwImgColumn, h.columns_off, h.num_columns)
            self._dir = (h, strings, tbytes, fields, terms, cols)
        return self._dir

    def field_names(self) -> List[str]:
        _h, strings, _tb, fields, _t, _c = self._directory()
        return [strings[f.name_off: f.name_off + f.name_len].decode() for f in fields]

    def column_names(self) -> List[str]:
        _h, strings, _tb, _f, _t, cols = self._directory()
        return [strings[c.name_off: c.name_off + c.name_len].decode() for c in cols]

    def columns(self):
        return self._directory()[5]

    def terms(self):
        return self._directory()[4]

    def fields(self):
        return self._directory()[3]

    def term_ord(self, field: str, term: bytes | str) -> int:
        """Dictionary lookup (test helper): ord of (field, term) or -1."""
        if isinstance(term, str):
            term = term.encode()
        _h, _s, tbytes, fields, terms, _c = self._directory()
        names = self.field_names()
        if field not in names:
            return -1
        f = fields[names.index(field)]
        for t in range(f.first_term, f.first_term + f.num_terms):
            if tbytes[terms[t].bytes_off: terms[t].bytes_off + terms[t].bytes_len] == term:
                return t
        return -1

    def column_ord(self, name: str) -> int:
        names = self.column_names()
        return names.index(name) if name in names else -1

    def doc_freq(self, term_ord: int) -> int:
        return self.terms()[term_ord].doc_freq

    def dictionary(self, column: int) -> List[bytes]:
        """Sorted term dictionary of a STR column."""
        h, strings, _tb, _f, _t, cols = self._directory()
        c = cols[column]
        n = c.dict_num_terms
        offs = struct.unpack_from(f"<{n + 1}I", strings, c.dict_off)
        base = c.dict_off + 4 * (n + 1)
        return [strings[base + offs[i]: base + offs[i + 1]] for i in range(n)]


# ---- value mappings (tantivy MonotonicallyMappableToU64) ---------------------------------------

def i64_to_u64(v: int) -> int:
    return (v + (1 << 63)) & 0xFFFFFFFFFFFFFFFF


def u64_to_i64(v: int) -> int:
    return ((v ^ (1 << 63)) & 0xFFFFFFFFFFFFFFFF) - (1 << 64) if (v ^ (1 << 63)) >> 63 else (v ^ (1 << 63))


def f64_to_u64(x: float) -> int:
    bits = struct.unpack("<Q", struct.pack("<d", x))[0]
    return (~bits) & 0xFFFFFFFFFFFFFFFF if bits >> 63 else bits ^ (1 << 63)


def u64_to_f64(v: int) -> float:
    bits = v ^ (1 << 63) if v >> 63 else (~v) & 0xFFFFFFFFFFFFFFFF
    return struct.unpack("<d", struct.pack("<Q", bits))[0]


def parse_datetime_nanos(v: Any) -> int:
    """rfc3339 string or unix timestamp (seconds; int or float) -> nanoseconds since epoch."""
    if isinstance(v, (int, np.integer)):
        return int(v) * 10**9
    if isinstance(v, float):
        return int(round(v * 10**9))
    s = str(v)
    if s.endswith("Z"):
        s = s[:-1] + "+00:00"
    d = _dt.datetime.fromisoformat(s)
    if d.tzinfo is None:
        d = d.replace(tzinfo=_dt.timezone.utc)
    epoch = _dt.datetime(1970, 1, 1, tzinfo=_dt.timezone.utc)
    delta = d - epoch
    return (delta.days * 86400 + delta.seconds) * 10**9 + delta.microseconds * 1000


# ---- tokenizers ----------------------------------------------------------------------------------

def decode_bytes_value(v: Any, input_format: str = "base64") -> bytes:
    """A `type: bytes` field value as the doc mapper reads it: a base64 (default) or hex string; bytes pass as is."""
    if isinstance(v, (bytes, bytearray)):
        return bytes(v)
    if input_format == "hex":
        return bytes.fromhex(str(v))
    if input_format == "base64":
        return base64.b64decode(str(v), validate=True)
    raise ValueError(f"unknown bytes input_format `{input_format}`")


def tokenize_default(text: str) -> List[str]:
    """tantivy "default" tokenizer (SimpleTokenizer + RemoveLong(255) + LowerCaser), restricted to
    ASCII case folding; any non-ASCII byte counts as a token character (same rule as the C++
    query-side tokenizer in query_compile.cpp)."""
    out, cur = [], []
    for ch in text:
        if (ch.isascii() and ch.isalnum()) or not ch.isascii():
            cur.append(ch.lower() if ch.isascii() else ch)
        elif cur:
            out.append("".join(cur))
            cur = []
    if cur:
        out.append("".join(cur))
    return [t for t in out if len(t.encode()) <= 255]


def tokenize(text: str, tokenizer: str) -> List[str]:
    return [text] if tokenizer == "raw" else tokenize_default(text)


# ---- builder -------------------------------------------------------------------------------------

class _Builder:
    def __init__(self, num_docs: int):
        self.L = ffi.img_lib()
        self.b = self.L.qwgpu_imgb_new(num_docs)
        self.num_docs = num_docs

    def add_field(self, name, flags, tok, fieldnorm_ids: Optional[np.ndarray], total_tokens: int) -> int:
        p = fieldnorm_ids.ctypes.data if fieldnorm_ids is not None else None
        return ffi.img_check(self.L.qwgpu_imgb_add_field(self.b, name.encode(), flags, tok, p, total_tokens))

    def add_term(self, field_id: int, term: bytes, docs: np.ndarray, tfs: Optional[np.ndarray], positions: Optional[np.ndarray] = None):
        docs = np.ascontiguousarray(docs, dtype=np.uint32)
        tfp = None
        if tfs is not None:
            tfs = np.ascontiguousarray(tfs, dtype=np.uint32)
            tfp = tfs.ctypes.data
        buf = C.create_string_buffer(term, len(term))
        if positions is not None:
            positions = np.ascontiguousarray(positions, dtype=np.uint32)
            ffi.img_check(self.L.qwgpu_imgb_add_term_positions(self.b, field_id, C.addressof(buf), len(term), docs.ctypes.data, tfp,
                                                               len(docs), positions.ctypes.data, len(positions)))
            return
        ffi.img_check(self.L.qwgpu_imgb_add_term(self.b, field_id, C.addressof(buf), len(term),
                                             docs.ctypes.data, tfp, len(docs)))

    def add_column(self, name: str, ctype: int, card: int, values: np.ndarray,
                   index: Optional[np.ndarray], dictionary: Optional[List[bytes]] = None):
        values = np.ascontiguousarray(values, dtype=np.uint64)
        ip = None
        if index is not None:
            index = np.ascontiguousarray(index, dtype=np.uint32)
            ip = index.ctypes.data
        dbytes = doffs = None
        dn = 0
        if dictionary is not None:
            dn = len(dictionary)
            blob = b"".join(dictionary)
            offs = np.zeros(dn + 1, dtype=np.uint32)
            np.cumsum([len(t) for t in dictionary], out=offs[1:])
            dbuf = C.create_string_buffer(blob, max(len(blob), 1))
            dbytes, doffs = C.addressof(dbuf), offs.ctypes.data
            self._keep = (dbuf, offs)
        ffi.img_check(self.L.qwgpu_imgb_add_column(self.b, name.encode(), ctype, card, values.ctypes.data,
                                               len(values), ip, dbytes, doffs, dn))

    def finish(self, split_id: str) -> SplitImage:
        out, n = C.c_void_p(), C.c_uint64()
        try:
            ffi.img_check(self.L.qwgpu_imgb_finish(self.b, C.byref(out), C.byref(n)))
        finally:
            self.L.qwgpu_imgb_free(self.b)
            self.b = None
        arr = np.frombuffer(ffi.take_bytes(out, n.value), dtype=np.uint8)
        return SplitImage(arr, split_id)


def _column_from_values(b: _Builder, name: str, ctype: int, per_doc: List[List[int]],
                        dictionary: Optional[List[bytes]] = None):
    """per_doc[d] = list of mapped-u64 values of doc d."""
    n = len(per_doc)
    counts = np.array([len(v) for v in per_doc], dtype=np.int64)
    flat = np.array([x for v in per_doc for x in v], dtype=np.uint64)
    if counts.size and counts.max(initial=0) <= 1:
        if counts.min(initial=1) == 1 and n > 0:
            b.add_column(name, ctype, ffi.CARD_FULL, flat, None, dictionary)
        else:
            b.add_column(name, ctype, ffi.CARD_OPTIONAL, flat, np.nonzero(counts)[0].astype(np.uint32), dictionary)
    else:
        start = np.zeros(n + 1, dtype=np.uint32)
        np.cumsum(counts, out=start[1:])
        b.add_column(name, ctype, ffi.CARD_MULTI, flat, start, dictionary)


_TYPE_TO_COL = {"u64": ffi.COL_U64, "i64": ffi.COL_I64, "f64": ffi.COL_F64, "bool": ffi.COL_BOOL,
                "datetime": ffi.COL_DATETIME}


def _map_value(ftype: str, v: Any, precision_ns: int = 1) -> int:
    if ftype == "u64":
        return int(v)
    if ftype == "i64":
        return i64_to_u64(int(v))
    if ftype == "f64":
        return f64_to_u64(float(v))
    if ftype == "bool":
        return 1 if v else 0
    if ftype == "datetime":
        ns = parse_datetime_nanos(v)
        ns -= ns % precision_ns  # DateTime::truncate(fast_precision)
        return i64_to_u64(ns)
    raise ValueError(ftype)


def build_split(docs: Sequence[Dict[str, Any]], doc_mapping: Dict[str, Any], split_id: str = "split") -> SplitImage:
    """Indexes `docs` (doc id = position) into one split image under `doc_mapping`."""
    n = len(docs)
    b = _Builder(n)
    mappings = {m["name"]: dict(m) for m in doc_mapping.get("field_mappings", [])}
    dynamic = doc_mapping.get("mode", "lenient") == "dynamic"
    if dynamic:
        dyn = doc_mapping.get("dynamic_mapping", {})
        for d in docs:
            for k, v in d.items():
                if k in mappings:
                    continue
                sample = v[0] if isinstance(v, list) and v else v
                if isinstance(sample, bool):
                    t = "bool"
                elif isinstance(sample, int):
                    t = "i64" if sample < 0 else "u64"
                elif isinstance(sample, float):
                    t = "f64"
                else:
                    t = "text"
                mappings[k] = {"name": k, "type": t, "fast": dyn.get("fast", True), "tokenizer": "raw",
                               "_dynamic": True}
        # numeric type coercion across docs (tantivy columnar: i64 > u64 > f64 preference)
        for k, m in mappings.items():
            if not m.get("_dynamic") or m["type"] not in ("u64", "i64", "f64"):
                continue
            vals = [x for d in docs if k in d for x in (d[k] if isinstance(d[k], list) else [d[k]])]
            if any(isinstance(x, float) for x in vals):
                m["type"] = "f64"
            elif any(isinstance(x, int) and x < 0 for x in vals):
                m["type"] = "i64"
            elif all(isinstance(x, int) and x < 2**63 for x in vals):
                m["type"] = "i64"
            else:
                m["type"] = "u64"
    for name, m in mappings.items():
        ftype = m.get("type", "text")
        values = [(d.get(name) if isinstance(d.get(name), list) else ([d[name]] if name in d and d[name] is not None else []))
                  for d in docs]
        if ftype == "text":
            tokenizer = m.get("tokenizer", "default")
            record = m.get("record", "basic")
            fieldnorms = bool(m.get("fieldnorms", False))
            if m.get("indexed", True):
                flags = (ffi.FIELD_HAS_FREQS if record in ("freq", "position") else 0) | \
                        (ffi.FIELD_HAS_FIELDNORMS if fieldnorms else 0) | (ffi.FIELD_HAS_POSITIONS if record == "position" else 0)
                postings: Dict[bytes, Dict[int, int]] = {}
                positions: Dict[bytes, Dict[int, List[int]]] = {}
                lengths = np.zeros(n, dtype=np.uint32)
                for d, vs in enumerate(values):
                    # token positions run across the values of a multi-valued field with a gap of one between
                    # values (tantivy postings_writer: end_position + POSITION_GAP)
                    start = 0
                    for v in vs:
                        toks = tokenize(str(v), tokenizer)
                        lengths[d] += len(toks)
                        for i, t in enumerate(toks):
                            postings.setdefault(t.encode(), {}).setdefault(d, 0)
                            postings[t.encode()][d] += 1
                            positions.setdefault(t.encode(), {}).setdefault(d, []).append(start + i)
                        start += len(toks) + 1
                L = ffi.img_lib()
                fn = np.array([L.qwgpu_fieldnorm_to_id(int(x)) for x in lengths], dtype=np.uint8) if fieldnorms else None
                fid = b.add_field(name, flags, ffi.TOK_RAW if tokenizer == "raw" else ffi.TOK_DEFAULT, fn, int(lengths.sum()))
                for term in sorted(postings):
                    dd = postings[term]
                    ds = np.array(sorted(dd), dtype=np.uint32)
                    tfs = np.array([dd[int(x)] for x in ds], dtype=np.uint32) if flags & ffi.FIELD_HAS_FREQS else None
                    pos = None
                    if flags & ffi.FIELD_HAS_POSITIONS:
                        pos = np.array([p for x in ds for p in positions[term][int(x)]], dtype=np.uint32)
                    b.add_term(fid, term, ds, tfs, pos)
            if m.get("fast", False):
                dictionary = sorted({str(v).encode() for vs in values for v in vs})
                ords = {t: i for i, t in enumerate(dictionary)}
                per_doc = [[ords[str(v).encode()] for v in vs] for vs in values]
                _column_from_values(b, name, ffi.COL_STR, per_doc, dictionary)
        elif ftype == "bytes":
            if m.get("fast", False):
                raw = [[decode_bytes_value(v, m.get("input_format", "base64")) for v in vs] for vs in values]
                dictionary = sorted({v for vs in raw for v in vs})
                ords = {t: i for i, t in enumerate(dictionary)}
                _column_from_values(b, name, ffi.COL_BYTES, [[ords[v] for v in vs] for vs in raw], dictionary)
        else:
            prec = _PRECISION_NS[m.get("fast_precision", "seconds")] if ftype == "datetime" else 1
            if m.get("fast", False) or m.get("_dynamic"):
                per_doc = [[_map_value(ftype, v, prec) for v in vs] for vs in values]
                _column_from_values(b, name, _TYPE_TO_COL[ftype], per_doc)
    return b.finish(split_id)


def synth_split(num_docs: int, split_ord: int, term_fracs: Iterable[float], seed: int = 0x5157,
                ts_start_secs: int = 1_700_000_000, ts_span_secs: int = 86_400, num_tenants: int = 100,
                split_id: Optional[str] = None, msg_vocab: int = 0) -> SplitImage:
    """Synthetic hdfs-logs-shaped split (SURVEY.md §8d); generation is done by the C++ writer.
    msg_vocab > 0 adds the text field "msg" with positions (phrase queries, BASELINE config 5)."""
    L = ffi.img_lib()
    fr = np.ascontiguousarray(list(term_fracs), dtype=np.float64)
    spec = ffi.SynthSpec(num_docs, split_ord, seed, len(fr), fr.ctypes.data_as(C.POINTER(C.c_double)),
                         ts_start_secs, ts_span_secs, num_tenants, msg_vocab, 0)
    out, n = C.c_void_p(), C.c_uint64()
    ffi.img_check(L.qwgpu_synth_split(C.byref(spec), C.byref(out), C.byref(n)))
    arr = np.ctypeslib.as_array(C.cast(out, C.POINTER(C.c_uint8)), shape=(n.value,)).copy()
    L.qwgpu_buf_free(out)
    return SplitImage(arr, split_id or f"split-{split_ord:04d}")
