"""Synthetic record tables for the BASELINE.json configurations (SURVEY.md section 8d).

gen(seed, N, dup, attrs, distortion, missing, F): N records over ~N*(1-dup) true entities; constant attributes
take Zipf-distributed values from a small vocabulary; Levenshtein attributes take strings from a vocabulary of
base strings (length 5-12 over a 26-letter alphabet, Zipf frequencies) plus 1-2-edit variants; a record's
attribute is distorted with probability `distortion` (string -> one of its base string's variants, constant ->
fresh draw) and missing with probability `missing`.  Deterministic in `seed` (numpy PCG64).
"""
from dataclasses import dataclass
from typing import List

import numpy as np

from .records import Attribute, SimilarityFn

ALPHABET = np.array(list("ABCDEFGHIJKLMNOPQRSTUVWXYZ"))


@dataclass
class SynthAttr:
    name: str
    kind: str  # "constant" | "levenshtein"
    vocab: int
    zipf: float = 1.0


def _zipf_probs(n, s):
    w = 1.0 / np.arange(1, n + 1) ** s
    return w / w.sum()


def _edit(rng, s):
    ops = rng.integers(1, 3)
    s = list(s)
    for _ in range(ops):
        op = rng.integers(0, 3)
        pos = rng.integers(0, max(len(s), 1))
        ch = ALPHABET[rng.integers(0, 26)]
        if op == 0 and len(s) > 0:
            s[pos] = ch
        elif op == 1:
            s.insert(pos, ch)
        elif len(s) > 3:
            del s[pos]
    return "".join(s)


def _string_vocab(rng, n_total):
    """n_total/4 base strings each followed by up to 3 distinct variants -> (strings, base_of[string])."""
    n_base = max(1, n_total // 4)
    strings, base_of, seen = [], [], set()
    for b in range(n_base):
        while True:
            ln = rng.integers(5, 13)
            s = "".join(ALPHABET[rng.integers(0, 26, ln)])
            if s not in seen:
                break
        seen.add(s)
        strings.append(s)
        base_of.append(b)
        for _ in range(3):
            v = _edit(rng, s)
            if v not in seen:
                seen.add(v)
                strings.append(v)
                base_of.append(b)
    return strings, np.array(base_of)


def config_attrs(config: int) -> List[SynthAttr]:
    if config == 3:  # 100k / 8 string attributes
        return [SynthAttr(f"s{i}", "levenshtein", 1000, 1.0) for i in range(8)]
    if config in (4, 5):  # 1M / 4 constant + 6 Levenshtein
        cs = [SynthAttr("c0", "constant", 100, 0.5), SynthAttr("c1", "constant", 12, 0.5),
              SynthAttr("c2", "constant", 31, 0.5), SynthAttr("c3", "constant", 50, 0.5)]
        z = 1.5 if config == 5 else 1.0
        return cs + [SynthAttr(f"s{i}", "levenshtein", 4000, z if i < 2 else 1.0) for i in range(6)]
    raise ValueError("config must be 3, 4 or 5")


def generate_encoded(seed, n_records, attrs: List[SynthAttr], dup=0.10, distortion=0.05, missing=0.01, n_files=1):
    """Array form: per attribute a vocabulary (list of strings) and a code per record (-1 = missing).
    -> dict(vocabs=[A][*] str, codes=int32[R, A], files=int32[R], ent_ids=int64[R], attributes=[Attribute],
    ent_values=int32[E, A]): ent_values[e] = the codes of entity e's true values, the values its records carry when
    not distorted (no random draw of its own: the other keys are those of the same seed without it)."""
    rng = np.random.default_rng(seed)
    R = int(n_records)
    n_ent = max(1, int(round(R * (1.0 - dup))))
    ent_of = np.concatenate([np.arange(n_ent), rng.integers(0, n_ent, R - n_ent)])
    rng.shuffle(ent_of)
    vocabs, codes = [], np.empty((R, len(attrs)), np.int32)
    ent_values = np.empty((n_ent, len(attrs)), np.int32)
    for a, sa in enumerate(attrs):
        if sa.kind == "constant":
            vocab = [f"{i:03d}" for i in range(sa.vocab)]
            p = _zipf_probs(sa.vocab, sa.zipf)
            ent_val = rng.choice(sa.vocab, n_ent, p=p)
            ent_values[:, a] = ent_val
            val = ent_val[ent_of]
            dist = rng.random(R) < distortion
            val = np.where(dist, rng.choice(sa.vocab, R, p=p), val)
        else:
            vocab, base_of = _string_vocab(rng, sa.vocab)
            base_idx = np.flatnonzero(np.r_[True, base_of[1:] != base_of[:-1]])  # first string of each base
            n_base = len(base_idx)
            p = _zipf_probs(n_base, sa.zipf)
            ent_base = rng.choice(n_base, n_ent, p=p)
            ent_values[:, a] = base_idx[ent_base]
            rec_base = ent_base[ent_of]
            first = base_idx[rec_base]
            count = np.r_[base_idx[1:], len(vocab)][rec_base] - first
            dist = rng.random(R) < distortion
            off = np.where(dist, rng.integers(0, 1 << 30, R) % np.maximum(count, 1), 0)
            val = first + off
        miss = rng.random(R) < missing
        codes[:, a] = np.where(miss, -1, val)
        vocabs.append(vocab)
    files = rng.integers(0, n_files, R).astype(np.int32) if n_files > 1 else np.zeros(R, np.int32)
    attributes = [
        Attribute(sa.name, SimilarityFn("ConstantSimilarityFn") if sa.kind == "constant"
                  else SimilarityFn("LevenshteinSimilarityFn", 7.0, 10.0), alpha=10.0, beta=1000.0)
        for sa in attrs
    ]
    return {"vocabs": vocabs, "codes": codes, "files": files, "ent_ids": ent_of, "attributes": attributes,
            "ent_values": ent_values}


def generate(seed, n_records, attrs: List[SynthAttr], dup=0.10, distortion=0.05, missing=0.01, n_files=1):
    """String form of generate_encoded:
    -> dict(values=[R][A] str|None, files=[R] str, rec_ids=[R] str, ent_ids=int[R], attributes=[Attribute])."""
    e = generate_encoded(seed, n_records, attrs, dup, distortion, missing, n_files)
    R = e["codes"].shape[0]
    cols = []
    for a, vocab in enumerate(e["vocabs"]):
        c = e["codes"][:, a]
        col = np.array(vocab + [None], dtype=object)[np.where(c < 0, len(vocab), c)].tolist()
        cols.append(col)
    values = [list(t) for t in zip(*cols)]
    return {"values": values, "files": [str(f) for f in e["files"]], "rec_ids": [str(i) for i in range(R)],
            "ent_ids": e["ent_ids"], "attributes": e["attributes"]}


def build_encoded(enc, expected_max_cluster_size=10):
    """RecordsCache.apply + transformRecords (RecordsCache.scala:68-133) on the array form: value counts by
    bincount, one AttributeIndex per attribute, codes remapped to sorted-string value ids.
    -> (indexes, x int32[R, A], file int32[R], num_files)"""
    from .engine import AttributeIndex

    codes = enc["codes"]
    R, A = codes.shape
    x = np.full((R, A), -1, np.int32)
    indexes = []
    for a, attr in enumerate(enc["attributes"]):
        vocab = enc["vocabs"][a]
        c = codes[:, a]
        cnt = np.bincount(c[c >= 0], minlength=len(vocab))
        used = np.flatnonzero(cnt)
        sf = attr.similarity_fn
        ix = AttributeIndex.build({vocab[i]: float(cnt[i]) for i in used}, sf.index_kind, sf.threshold,
                                  sf.max_similarity, expected_max_cluster_size)
        lut = np.full(len(vocab) + 1, -1, np.int32)
        for i in used:
            lut[i] = ix.value_idx_of(vocab[i])
        x[:, a] = lut[np.where(c < 0, len(vocab), c)]
        indexes.append(ix)
    files = enc["files"]
    return indexes, x, np.ascontiguousarray(files, np.int32), int(files.max()) + 1
