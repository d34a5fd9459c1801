"""Long-phrase restatements for the tests: the per-term postings of a list of documents, positioned the way
splitgen.build_split indexes them (the arrays scoring_ref.phrase_counts reads), phrases cut from documents, and the
f32 score a phrase count gives."""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Sequence

import numpy as np

from quickwit_b200 import ffi, splitgen as S
from helpers import bm25_norm
from phrase_prefix_ref import doc_positions


def values_of(doc: Dict, field: str) -> List[str]:
    v = doc.get(field)
    return [] if v is None else (v if isinstance(v, list) else [v])


class TokenPostings:
    """`postings[(field, token)]` = (docs, tfs, positions) of `docs`, and each doc's token count (its fieldnorm)."""

    def __init__(self, docs: Sequence[Dict], field: str):
        self.n = len(docs)
        self.lengths = np.zeros(self.n, dtype=np.int64)
        per: Dict[str, list] = {}
        for d, doc in enumerate(docs):
            vals = values_of(doc, field)
            self.lengths[d] = sum(len(S.tokenize_default(v)) for v in vals)
            for t, ps in doc_positions(vals).items():
                per.setdefault(t, []).append((d, ps))
        self.postings = {}
        for t, rows in per.items():
            self.postings[(field, t)] = (np.array([d for d, _ in rows], dtype=np.uint32),
                                         np.array([len(p) for _, p in rows], dtype=np.uint32),
                                         np.array([x for _, p in rows for x in p], dtype=np.uint32))


def phrase_ast(field: str, text: str, mode: str = "phrase"):
    return {"type": "full_text", "field": field, "text": text, "params": {"mode": {"type": mode, "slop": 0}},
            "lenient": False}


def windows(tokens: Sequence[str], lo: int, hi: int) -> List[List[str]]:
    """Every window of lo..hi tokens."""
    return [list(tokens[s:s + n]) for n in range(lo, hi + 1) for s in range(len(tokens) - n + 1)]


def phrase_weight(img, field: str, tokens: Sequence[str], boost: float = 1.0) -> np.float32:
    """Bm25Weight::for_terms through the library (the weight a hand-built plan carries)."""
    dfs = [img.doc_freq(img.term_ord(field, t)) for t in tokens]
    arr = (C.c_uint64 * len(dfs))(*dfs)
    return np.float32(ffi.img_lib().qwgpu_bm25_phrase_weight(arr, len(dfs), img.num_docs, boost))


def expected_scores(img, field: str, counts: np.ndarray, docs: np.ndarray, lengths: np.ndarray, weight,
                    fieldnorms: bool) -> np.ndarray:
    """weight * (count / (count + norm)) in f32: norm from the docs' quantised token counts, or, for a field without
    fieldnorms, the constant norm of a length-1 doc against the field's average length."""
    f32 = np.float32
    if fieldnorms:
        norm = bm25_norm(lengths)[docs]
    else:
        fld = img.fields()[img.field_names().index(field)]
        avg = f32(fld.total_num_tokens) / f32(img.num_docs)
        norm = np.full(len(docs), f32(1.2) * (f32(1) - f32(0.75) + f32(0.75) * f32(1) / avg), dtype=np.float32)
    tf = counts.astype(np.float32)
    return (f32(weight) * (tf / (tf + norm))).astype(np.float32)
