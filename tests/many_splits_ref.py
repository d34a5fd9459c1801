"""Leaf requests over many splits: the base images, the ids they are registered under, and a brute force of the leaf
merge over every document of every split.

A base image is registered under many split ids. Twins tie on every sort value (f32 scores included), so their hits
are ordered by (split id, doc id) alone. The brute force restates the merge (collector.rs:1120-1153): sort values
with None last in both directions, then (split id, doc id) in the direction of the first key. It reads each base's
matches and column values from the image, and for `_score` sorts the oracle's complete per-split hit list (f32
scores); it shares no code with the product's merge."""
import json
import numpy as np

from quickwit_b200 import ffi, proto, splitgen as S
from quickwit_b200.proto import ASC, DESC
from oracle import oracle as O
from pipeline import search_request

T0 = 1_700_000_000
DAY = 86_400
MAPPING = {"field_mappings": [{"name": "body", "type": "text", "record": "freq", "fieldnorms": True},
                              {"name": "severity_text", "type": "text", "tokenizer": "raw", "fast": True},
                              {"name": "timestamp", "type": "datetime", "fast": True, "fast_precision": "seconds"},
                              {"name": "tenant_id", "type": "u64", "fast": True},
                              {"name": "c", "type": "u64", "fast": True}], "timestamp_field": "timestamp"}
DM = json.dumps(MAPPING)
SYNTH_FRACS = [0.2, 0.1, 0.05, 0.02, 0.01]
# k_union's window is 15 360 docs: the hand-made shapes sit on either side of one window and of a posting block
HAND_DOCS = (0, 1, 127, 15_359, 15_360, 15_361, 40_000)


def hand_split(n, seed, split_id="hand", with_c=True, solo=False):
    """A split built from numpy arrays: body terms t0 (every doc, tf 1..7), t1 (one doc in 9), t2 (one doc in 4001),
    `solo` (one doc in 50, only when asked for); severity_text; a timestamp inside [T0, T0 + DAY); tenant_id with
    13 values; and the optional column c (50 values, about one doc in five without it) unless with_c is False."""
    d = np.arange(n, dtype=np.int64)
    b = S._Builder(n)
    lens = 3 + (d * 7 + seed) % 11
    L = ffi.img_lib()
    fn = np.array([L.qwgpu_fieldnorm_to_id(int(x)) for x in range(64)], dtype=np.uint8)[lens] if n else np.zeros(0, np.uint8)
    body = b.add_field("body", ffi.FIELD_HAS_FREQS | ffi.FIELD_HAS_FIELDNORMS, ffi.TOK_DEFAULT, fn, int(lens.sum()))
    terms = {b"t0": (d, 1 + (d * 5 + seed) % 7), b"t1": (d[d % 9 == seed % 9], None), b"t2": (d[d % 4001 == 17], None)}
    if solo:
        terms[b"solo"] = (d[d % 50 == 3], None)
    for t in sorted(terms):
        docs, tf = terms[t]
        b.add_term(body, t, docs, tf if tf is not None else np.ones(len(docs), np.uint32))
    sev = (d * 31 + seed) % 4
    sf = b.add_field("severity_text", 0, ffi.TOK_RAW, None, n)
    names = [b"DEBUG", b"ERROR", b"INFO", b"WARN"]
    for o, name in enumerate(names):
        b.add_term(sf, name, d[sev == o], None)
    b.add_column("severity_text", ffi.COL_STR, ffi.CARD_FULL, sev.astype(np.uint64), None, names)
    ts = (T0 + (d * 37 + seed) % DAY) * 10**9
    b.add_column("timestamp", ffi.COL_DATETIME, ffi.CARD_FULL, ts.astype(np.uint64) ^ np.uint64(1 << 63), None)
    b.add_column("tenant_id", ffi.COL_U64, ffi.CARD_FULL, ((d * 3 + seed) % 13).astype(np.uint64), None)
    if with_c:
        has = np.flatnonzero((d * 2654435761 + seed) % 5 != 0).astype(np.uint32)
        b.add_column("c", ffi.COL_U64, ffi.CARD_OPTIONAL, ((has.astype(np.int64) * 7919 + seed) % 50).astype(np.uint64), has)
    return b.finish(split_id)


def synth(ordinal, n):
    """A synthetic split whose timestamps cover day `ordinal` after T0 + DAY: every such split's range is disjoint from
    every other's and from the hand-made splits'. It has no column c."""
    return S.synth_split(n, 1000 + ordinal, SYNTH_FRACS, ts_start_secs=T0 + DAY * (1 + ordinal), ts_span_secs=DAY,
                         split_id=f"synth-base-{ordinal}")


def ids(prefix, count, seed):
    """[(i, split id)] for i < count, shuffled. The ids' lexical order differs from their numeric order (`p-7` sorts
    after `p-10`), and id i is the same at every count."""
    rng = np.random.default_rng(seed)
    return [(int(i), f"{prefix}-{i}" if i % 3 else f"{prefix}{i % 7}-{i}") for i in rng.permutation(count)]


class Base:
    """One base image and what the brute force reads from it, cached."""

    def __init__(self, img):
        self.img = img
        self.n = img.num_docs
        self._cols, self._match = {}, {}

    def column(self, name):
        """(mapped u64 values, present) of the column's first value per doc; all absent when the split lacks it."""
        if name not in self._cols:
            if name in self.img.column_names():
                self._cols[name] = O.column_first(self.img, self.img.column_ord(name))
            else:
                self._cols[name] = (np.zeros(self.n, np.uint64), np.zeros(self.n, bool))
        return self._cols[name]

    def matches(self, ast):
        """Docs matching a match_all or single-term query."""
        key = json.dumps(ast, sort_keys=True)
        if key not in self._match:
            if ast["type"] == "match_all":
                m = np.arange(self.n, dtype=np.int64)
            else:
                assert ast["type"] == "term", ast
                try:
                    t = self.img.term_ord(ast["field"], ast["value"])
                except (KeyError, ValueError):
                    t = -1
                m = O.decode_postings(self.img, t, self.n)[0].astype(np.int64) if t >= 0 else np.zeros(0, np.int64)
            self._match[key] = m
        return self._match[key]

    def scores(self, ast, order):
        """Every matching doc with its f32 score: the oracle's complete hit list of the split."""
        key = ("score", json.dumps(ast, sort_keys=True), order)
        if key not in self._match:
            from quickwit_b200 import service
            req = search_request(ast, max_hits=max(self.n, 1), sort_fields=[("_score", order)])
            r = O.split_search(self.img, service.compile_plan(self.img, req, DM))
            assert len(r.hits) == r.num_hits
            self._match[key] = (np.array([h[0] for h in r.hits], np.int64), np.array([h[4] for h in r.hits], np.float32))
        return self._match[key]


FIELD_TYPE = {"tenant_id": "u64", "c": "u64", "timestamp": "datetime"}


def typed(field, v):
    if FIELD_TYPE[field] == "u64":
        return ("u64", int(v))
    return ("i64", S.u64_to_i64(int(v)))


def in_time_range(base, docs, start, end):
    """Docs whose timestamp (seconds) lies in [start, end): the request's start_timestamp / end_timestamp."""
    v, has = base.column("timestamp")
    secs = (v[docs] ^ np.uint64(1 << 63)).astype(np.int64) // 10**9
    return has[docs] & (secs >= start) & (secs < end)


def _keys(base, ast, sort, time_range=None):
    """Per-doc sort keys of the split's matches: (docs, [(has, value key ascending = better first)], typed values)."""
    if sort[0][0] == "_score":
        docs, sc = base.scores(ast, sort[0][1])
        key = (-sc.astype(np.float64)) if sort[0][1] == DESC else sc.astype(np.float64)
        return docs, [(np.ones(len(docs), bool), key)], [("f64", float(x)) for x in sc]
    docs = base.matches(ast)
    if time_range is not None:
        docs = docs[in_time_range(base, docs, *time_range)]
    if sort[0][0] == "_doc":
        return docs, [], None
    keys, vals = [], []
    for field, order in sort:
        v, has = base.column(field)
        v, has = v[docs], has[docs]
        k = np.where(has, ~v if order == DESC else v, np.uint64(0))
        keys.append((has, k))
        vals.append((v, has))
    return docs, keys, vals


def expected(entries, ast, sort, K, time_range=None):
    """The merged top K of a leaf request over `entries` = [(split id, Base)] (request order), as
    (num_hits, [(split id, doc id, sort_value, sort_value2)]); sort_value is None for a missing value."""
    names = sorted(e[0] for e in entries)
    rank = {s: i for i, s in enumerate(names)}
    desc = sort[0][1] == DESC
    parts, num_hits = [], 0
    cache = {}
    for sid, base in entries:
        if id(base) not in cache:
            docs, keys, vals = _keys(base, ast, sort, time_range)
            # the split's own order: keys, then doc id in the direction of the first key
            lk = [(-docs if desc else docs)]
            for has, k in reversed(keys):
                lk += [k, ~has]
            order = np.lexsort(lk) if len(docs) else np.zeros(0, np.int64)
            cache[id(base)] = (docs, keys, vals, order)
        docs, keys, vals, order = cache[id(base)]
        num_hits += len(docs)
        top = order[:K]
        parts.append((rank[sid], sid, docs, keys, vals, top))
    if K == 0 or not parts:
        return num_hits, []
    r = np.concatenate([np.full(len(p[5]), p[0], np.int64) for p in parts])
    d = np.concatenate([p[2][p[5]] for p in parts])
    pos = np.concatenate([np.arange(len(p[5])) for p in parts])
    src = np.concatenate([np.full(len(p[5]), i, np.int64) for i, p in enumerate(parts)])
    lk = [(-d if desc else d), (-r if desc else r)]
    for j in reversed(range(len(parts[0][3]))):
        lk += [np.concatenate([p[3][j][1][p[5]] for p in parts]), ~np.concatenate([p[3][j][0][p[5]] for p in parts])]
    sel = np.lexsort(lk)[:K]
    out = []
    for g in sel:
        p = parts[src[g]]
        i = p[5][pos[g]]
        sv = [None, None]
        if sort[0][0] == "_score":
            sv[0] = p[4][i]
        elif sort[0][0] != "_doc":
            for j, (field, _) in enumerate(sort):
                v, has = p[4][j]
                sv[j] = typed(field, v[i]) if has[i] else None
        out.append((p[1], int(d[g]), sv[0], sv[1]))
    return num_hits, out


def hits_of(resp):
    return [(h["split_id"], h["doc_id"], h.get("sort_value"), h.get("sort_value2")) for h in resp["partial_hits"]]


def leaf_request(entries, ast, sort, max_hits, start=0, **kw):
    """The leaf request for `entries` (root.rs:1775-1777: start_offset folded into max_hits) and the root request."""
    leaf = search_request(ast, max_hits=max_hits + start, start_offset=0, sort_fields=list(sort), **kw)
    root = search_request(ast, max_hits=max_hits, start_offset=start, sort_fields=list(sort), **kw)
    offsets = [proto.enc_split_offsets(sid, base.n) for sid, base in entries]
    return proto.enc_leaf_search_request(leaf, offsets, DM), root


def check_aggs(a, bases):
    """The finalized JSON of AGGS over splits `bases` (one per split id) against counts computed from the documents:
    severity buckets with their tenant sub-buckets, day buckets of the timestamp, and stats of tenant_id."""
    sev, days, ten = {}, {}, []
    for b in bases:
        if not b.n:
            continue
        s, _ = b.column("severity_text")
        names = [x.decode() for x in b.img.dictionary(b.img.column_ord("severity_text"))]
        t, _ = b.column("tenant_id")
        ts, _ = b.column("timestamp")
        day = ((ts ^ np.uint64(1 << 63)).astype(np.int64) // 10**9 // DAY) * DAY * 1000
        for o, name in enumerate(names):
            sub = sev.setdefault(name, {})
            for v, c in zip(*np.unique(t[s == o], return_counts=True)):
                sub[int(v)] = sub.get(int(v), 0) + int(c)
        for k, c in zip(*np.unique(day, return_counts=True)):
            days[int(k)] = days.get(int(k), 0) + int(c)
        ten.append(t.astype(np.int64))
    got = {bk["key"]: (bk["doc_count"], {int(x["key"]): x["doc_count"] for x in bk["ten"]["buckets"]}) for bk in a["sev"]["buckets"]}
    want = {k: (sum(v.values()), v) for k, v in sev.items() if v}
    assert got == want
    gd = {int(bk["key"]): bk["doc_count"] for bk in a["days"]["buckets"]}
    assert {k: v for k, v in gd.items() if v} == days and sum(gd.values()) == sum(days.values())
    t = np.concatenate(ten)
    st = a["ten"]
    assert (st["count"], st["min"], st["max"], st["sum"]) == (len(t), float(t.min()), float(t.max()), float(t.sum()))
    assert st["avg"] == float(t.sum()) / len(t)
