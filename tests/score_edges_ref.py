"""The level-0 `_score` bucket of the composite top-K key, restated in numpy float32 (DESIGN.md §4.6), and corpora whose
scores sit exactly on its edges.

A `_score` plan ranks a doc by a key whose first field is [1 | lin:10 | ordered f32 score:32], then the doc id in the
direction of the first key. lin = min(1023, floor(fmul_rn(score, score_scale))), score_scale = 1024 / score_max, and
score_max is the f32 sum of the plan's positive weights in lowering order. Every route reads that bucket in its own way:
k_union's sample histogram (`score_digit`) and float bound (`thresh_s_lo`), k_window's fast-path bound (bucket 0 filters
nothing there), `key_top11` / `score_lin` in rank_hist / rank_collect and `doc_key`. numpy's float32 `*` and `/` round
to nearest, like `__fmul_rn` / `__fdiv_rn` under -fmad=false (csrc/Makefile); nothing here reads the engine's code.

A corpus plants, per edge term, docs whose x = fmul(score, scale) is exactly an integer l, 1..8 ulps above it (inside
the ±1e-6 relative band that the bound's ×0.999999 factor leaves), 1..8 ulps below it (bucket l - 1), and a mass deeper
in bucket l - 1. Each edge term T is queried as `T OR tune_T`: tune_T holds one doc, and T's boost is searched so that
the asymptote fmul(w_T, scale) (a doc at tf -> inf) lies just above l, where consecutive tfs step x by less than one ulp
and every ulp near l is reachable."""
from __future__ import annotations

import numpy as np

from quickwit_b200 import ffi, plan as P, splitgen as S
from helpers import bm25_contributions, bm25_norm, bm25_weight

F32 = np.float32
BAND = 8                 # ulps on either side of an edge
TF_MAX = 0xFFFFFFFF      # the tf factor of this tf rounds to 1.0: the doc scores the term's whole weight


# ---- the key, restated -----------------------------------------------------------------------------------------------
def score_scale(weights) -> np.float32:
    """1024 / score_max: the f32 sum of the positive weights in lowering order (1.0 when it is not above 1e-30)."""
    smax = F32(0)
    for w in weights:
        w = F32(w)
        if w > 0:
            smax = F32(smax + w)
    if not smax > F32(1e-30):
        smax = F32(1)
    return F32(F32(1024) / smax)


def fmul(a, b):
    return (np.asarray(a, dtype=F32) * F32(b)).astype(F32)


def lin(s, scale, desc=True):
    """score_lin: the 10-bit bucket of the score, clamped at 1023, mirrored for ASC."""
    x = fmul(s, scale)
    l = np.where(x >= F32(1023), 1023, np.where(x > 0, np.floor(np.where(x > 0, x, 0)), 0)).astype(np.int64)
    return l if desc else 1023 - l


def digit(s, scale, desc=True):
    """The level-0 radix digit (the key's first 11 bits): [1 | lin:10]."""
    return 1024 | lin(s, scale, desc)


def s_lo_union(l, scale) -> np.float32:
    """k_union's f32 lower bound of bucket l (thresh_s_lo)."""
    return F32(F32(F32(l) / F32(scale)) * F32(0.999999))


def s_lo_window(l, scale) -> np.float32:
    """k_window's fast-path bound: the same, except that bucket 0 filters nothing."""
    return F32(-np.inf) if l == 0 else s_lo_union(l, scale)


def passes_union(s, l, scale):
    """A doc reaches k_union's candidate test for a threshold in bucket l."""
    s = np.asarray(s, dtype=F32)
    return (s > 0) & (s >= s_lo_union(l, scale))


def passes_window(s, l, scale):
    return np.asarray(s, dtype=F32) >= s_lo_window(l, scale)


def f32_ordered(s):
    b = np.asarray(s, dtype=F32).view(np.uint32).astype(np.uint64)
    return np.where(b >> np.uint64(31), ~b & np.uint64(0xFFFFFFFF), b | np.uint64(0x80000000))


def score_field(s, scale, desc=True):
    """The 42-bit score field of the key: [lin:10 | ordered f32:32], both mirrored for ASC."""
    o = f32_ordered(s)
    r = o if desc else ~o & np.uint64(0xFFFFFFFF)
    return (lin(s, scale, desc).astype(np.uint64) << np.uint64(32)) | r


def keys(s, docs, scale, doc_bits, desc=True):
    """The narrow composite key of a `_score`-only sort: [1 | score field:42 | doc:doc_bits], the doc id mirrored
    with the first key's order. Larger is better."""
    d = np.asarray(docs, dtype=np.uint64)
    docr = d if desc else np.uint64((1 << doc_bits) - 1) - d
    return (np.uint64(1) << np.uint64(42 + doc_bits)) | (score_field(s, scale, desc) << np.uint64(doc_bits)) | docr


def ulps_from(x, l):
    """Signed distance of f32 x from the integer l, in units in the last place."""
    return np.asarray(x, dtype=F32).view(np.int32).astype(np.int64) - int(F32(l).view(np.int32))


def rounds_up(s, scale):
    """x = fmul_rn(s, scale) rounded the exact product up (the f64 product of two f32 is exact)."""
    return np.asarray(s, dtype=np.float64) * float(scale) < fmul(s, scale).astype(np.float64)


def brute_order(s, matched, desc=True):
    """Matched doc ids in rank order: score (f32 bits), then the doc id in the same direction."""
    d = np.flatnonzero(matched)
    sc = np.asarray(s, dtype=F32)[d]
    return d[np.lexsort((-d, -sc))] if desc else d[np.lexsort((d, sc))]


def _nearest(u, want):
    """Index of a tf whose x is `want` ulps from the edge; else one exactly on it; else the closest to `want`."""
    for w in (want, 0):
        hit = np.flatnonzero(u == w)
        if len(hit):
            return hit[0]
    return np.argmin(np.abs(u - want))


# ---- corpora ---------------------------------------------------------------------------------------------------------
# per edge term: (docs per ulp above l, exact tie at l, docs per ulp below l, mass deeper in bucket l - 1)
EDGE_TERMS = {
    "e1": (4, 1500, 4, 9000),       # K = 1: the top doc is 8 ulps above the edge
    "e10": (0, 2000, 4, 9000),      # K = 10: inside the tie on the edge (four docs 1..4 ulps above it, see ABOVE_E10)
    "e1000": (50, 590, 100, 2000),  # K = 1000: 1..8 ulps below the edge
    "e4096": (12, 4500, 4, 0),      # K = 4096 / 4097: inside the tie on the edge
}
ABOVE_E10 = 4
EDGE_L = {"e1": 600, "e10": 520, "e1000": 280, "e4096": 560, "asc": 540}   # (just above a power of two: two f32 tf factors per ulp of x)
ASC = (40, 2000, 40, 3000)          # `_score` ASC: the lowest scores 1..8 ulps below the edge, then the tie on it
N_TOP = 120                         # docs of `top` near and in the clamped bucket 1023
CLAMP = (4000, 40, 9000)            # `ca OR cb`: docs at score_max (x = 1024), docs around x = 1023, one tie far below
G_EVERY = 8                         # `g`, the low-weight union companion: on one doc in 8
HEAD = 1024


class EdgeCorpus:
    """One split built from arrays: term frequencies per term (0 = absent), doc lengths, column f. `planted[T]` maps a
    class name ("above", "exact", "below", "mass") to its doc ids; `boost[T]` is the boost of T's plan clause."""

    def __init__(self, n, split_id, seed=7):
        self.n = n
        rng = np.random.default_rng(seed)
        d = np.arange(n, dtype=np.int64)
        # two docs of every planted class lie in the first HEAD docs, which every sample reads (window 0 of the split at
        # batch position 0, at every window size); the rest are spread over the split (a larger share there would
        # inflate the sampled counts of the planted buckets)
        head, free = rng.permutation(HEAD), HEAD + rng.permutation(n - HEAD)
        used = []

        def take(k):
            nonlocal head, free
            nh = min(2, k // 2)
            out = np.concatenate([head[:nh], free[: k - nh]])
            head, free = head[nh:], free[k - nh:]
            used.append(out)
            return np.sort(out)

        self.lens = 6 + (d * 7919) % 251            # every fieldnorm id from 6 to 256 tokens
        self.planted, self.boost, self.l = {}, {}, {}
        self.tf = {}
        layouts = dict(EDGE_TERMS, asc=ASC)
        pos = {}
        for t, (pa, ne, pb, nm) in layouts.items():
            na = ABOVE_E10 if t == "e10" else BAND * pa
            pos[t] = {"above": take(na), "exact": take(ne), "below": take(BAND * pb), "mass": take(nm)}
            pos["tune_" + t] = {"one": take(1)}
        pos["top"] = {"near": take(N_TOP), "max": take(N_TOP)}
        nmax, nnear, nmass = CLAMP
        pos["ca"] = {"max": take(nmax), "near": take(nnear), "mass": take(nmass)}
        pos["cb"] = {"max": pos["ca"]["max"], "near": pos["ca"]["near"]}
        pos["g"] = {"all": np.setdiff1d(d[d % G_EVERY == 3], np.concatenate(used))}
        pos["x"] = {"all": np.setdiff1d(d[d % 16 == 5], np.concatenate(used))}   # must_not: never a planted doc
        self.f = (d % 10).astype(np.uint64)
        self.f[np.concatenate([pos["top"]["near"], pos["top"]["max"]])] = 0   # the driver's range filter keeps `top`
        # every doc of one tie has one length: one score
        for t in layouts:
            self.lens[pos[t]["exact"]] = 40
        self.lens[pos["ca"]["mass"]] = 40
        self.norm = bm25_norm(self.lens)
        self.df = {t: sum(len(v) for v in c.values()) for t, c in pos.items()}
        for t, c in pos.items():
            self.tf[t] = np.zeros(n, dtype=np.int64)
            self.planted[t] = c
        self.tf["g"][pos["g"]["all"]] = 1 + pos["g"]["all"] % 3
        self.tf["x"][pos["x"]["all"]] = 1
        for t in layouts:
            self.tf["tune_" + t][pos["tune_" + t]["one"]] = 1
            self._plant(t, EDGE_L[t], pos[t])
        self._plant_top(pos["top"])
        self._plant_clamp(pos["ca"])
        self.img = self._build(split_id)

    # weights ------------------------------------------------------------------------------------------------------------
    def weight(self, t, boost=1.0):
        """The f32 weight the library compiles for term t (checked against the numpy restatement of idf)."""
        w = F32(P.bm25_weight(self.df[t], self.n, boost))
        want = F32(bm25_weight(self.df[t], self.n) * F32(boost))
        assert abs(float(w) - float(want)) <= 2e-6 * abs(float(want)), (t, w, want)
        return w

    def plan_weights(self, t):
        """(w_T, w_tune_T) of the plan `T OR tune_T`."""
        return self.weight(t, self.boost[t]), self.weight("tune_" + t)

    def scale(self, terms_boosts):
        return score_scale([self.weight(t, b) for t, b in terms_boosts])

    def scores(self, terms_boosts):
        """Union of the (term, boost) clauses in clause order, numpy float32."""
        s = np.zeros(self.n, dtype=F32)
        for t, b in terms_boosts:
            s = (s + bm25_contributions(self.tf[t], self.norm, self.weight(t, b))).astype(F32)
        return s

    def clauses(self, t):
        return [(t, self.boost[t]), ("tune_" + t, 1.0)]

    # planting ---------------------------------------------------------------------------------------------------------
    def _plant(self, t, l, pos):
        """Find T's boost (asymptote just above l) and a tf per planted doc for its class; a boost under which some
        class has no tf is passed over."""
        wt = self.weight("tune_" + t)
        b0 = float(wt) * (l + 0.01) / (1024 - l - 0.01) / float(self.weight(t))   # asymptote near l + 0.01
        for k in range(-30000, 30000):
            b = float(F32(b0 * (1 + 2e-7 * k)))
            w = F32(P.bm25_weight(self.df[t], self.n, b))
            a = float(fmul(w, score_scale([w, wt])))
            if l + 0.004 < a < l + 0.02:
                tf = self._plant_at(t, l, pos, w, score_scale([w, wt]), a)
                if tf is not None:
                    self.boost[t], self.l[t], self.tf[t] = b, l, tf
                    return
        raise AssertionError(f"no boost puts every class of {t} on its edge")

    def _plant_at(self, t, l, pos, w, scale, a):
        ulp = float(np.spacing(F32(l)))
        cache = {}

        def window(norm):
            """(tfs, x) over every tf whose x lies within 12 ulps of l (x rises with tf; tf(x) = norm x / (a - x))."""
            if norm not in cache:
                lo = max(1, int(norm * (l - 12 * ulp) / (a - l + 12 * ulp) * 0.99))
                hi = int(norm * (l + 12 * ulp) / (a - l - 12 * ulp) * 1.01) + 2
                tfs = np.arange(lo, hi, dtype=np.int64)
                cache[norm] = (tfs, fmul(bm25_contributions(tfs, F32(norm), w), scale))
            return cache[norm]

        def pick(doc, want_ulps, rz=False):
            norm = float(self.norm[doc])
            tfs, x = window(norm)
            hit = np.flatnonzero(ulps_from(x, l) == want_ulps)
            if rz:
                hit = hit[rounds_up(bm25_contributions(tfs[hit], F32(norm), w), scale)]
            return int(tfs[hit[len(hit) // 2]]) if len(hit) else None

        tf = np.zeros(self.n, dtype=np.int64)
        ex = pos["exact"]
        if len(ex):
            v = pick(int(ex[0]), 0, rz=True)
            if v is None:
                return None
            tf[ex] = v
        for cls, sign in (("above", 1), ("below", -1)):
            for i, doc in enumerate(pos[cls]):
                v = pick(int(doc), sign * (1 + i % BAND))
                if v is None:
                    return None
                tf[doc] = v
        # the mass lies deeper in the bucket below the edge (ASC: between the edge band and the asymptote)
        target = (l - 0.5) if t != "asc" else (l + a) / 2
        m = pos["mass"]
        tf[m] = np.maximum(1, np.rint(self.norm[m].astype(np.float64) * target / (a - target))).astype(np.int64)
        return tf

    def _plant_top(self, pos):
        """`top` alone is scored by the driver plan (score_max = its weight): tf max scores the whole weight, and x is
        1024 or just below it, in the clamped bucket 1023; the other docs sit on both sides of x = 1023."""
        w = self.weight("top")
        scale = score_scale([w])
        tf = self.tf["top"]
        tf[pos["max"]] = TF_MAX
        tfs = np.arange(1, 1 << 16, dtype=np.int64)
        for i, doc in enumerate(pos["near"]):
            x = fmul(bm25_contributions(tfs, self.norm[doc], w), scale)
            u = ulps_from(x, 1023)
            want = (i % (2 * BAND + 1)) - BAND                    # -8 .. 8 ulps around 1023
            tf[doc] = int(tfs[_nearest(u, want)])

    def _plant_clamp(self, pos):
        """`ca OR cb`, both clauses at tf 2^32 - 1: the doc scores exactly score_max, and ca's boost is searched so that
        x = fmul(score_max, scale) is 1024, the value only the clamp keeps in bucket 1023. Docs with ca at tf max and cb
        at a picked tf sit around x = 1023; one tie of ca alone sits far below, in a single bucket."""
        wb = self.weight("cb")
        for k in range(20000):
            b = float(F32(1.0 + 1e-6 * k))
            wa = F32(P.bm25_weight(self.df["ca"], self.n, b))
            scale = score_scale([wa, wb])
            if fmul(F32(wa + wb), scale) == F32(1024):
                break
        else:
            raise AssertionError("no boost of ca puts score_max at x = 1024")
        self.boost["ca"] = b
        ta, tb = self.tf["ca"], self.tf["cb"]
        ta[pos["max"]] = tb[pos["max"]] = TF_MAX
        ta[pos["near"]] = TF_MAX
        tfs = np.arange(1, 1 << 18, dtype=np.int64)
        for i, doc in enumerate(pos["near"]):
            s = (wa + bm25_contributions(tfs, self.norm[doc], wb)).astype(F32)
            u = ulps_from(fmul(s, scale), 1023)
            want = (i % (2 * BAND + 1)) - BAND                    # -8 .. 8 ulps around 1023
            tb[doc] = int(tfs[_nearest(u, want)])
        a = float(fmul(wa, scale))                                # ca alone at tf -> inf
        target = np.floor(0.8 * a) + 0.5
        m = pos["mass"]
        ta[m] = max(1, int(round(float(self.norm[m[0]]) * target / (a - target))))

    def clamp_clauses(self):
        return [("ca", self.boost["ca"]), ("cb", 1.0)]

    def _build(self, split_id):
        b = S._Builder(self.n)
        L = ffi.img_lib()
        uniq, inv = np.unique(self.lens, return_inverse=True)
        fn = np.array([L.qwgpu_fieldnorm_to_id(int(x)) for x in uniq], dtype=np.uint8)[inv]
        body = b.add_field("body", ffi.FIELD_HAS_FREQS | ffi.FIELD_HAS_FIELDNORMS, ffi.TOK_DEFAULT, fn, int(self.lens.sum()))
        for name in sorted(self.tf):
            docs = np.flatnonzero(self.tf[name]).astype(np.uint32)
            assert len(docs) == self.df[name], name
            b.add_term(body, name.encode(), docs, self.tf[name][docs].astype(np.uint32))
        b.add_column("f", ffi.COL_U64, ffi.CARD_FULL, self.f, None)
        return b.finish(split_id)

    def under_id(self, split_id):
        c = EdgeCorpus.__new__(EdgeCorpus)
        c.__dict__.update(self.__dict__)
        c.img = S.SplitImage(self.img.array, split_id)
        return c
