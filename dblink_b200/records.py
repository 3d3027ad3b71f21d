"""RecordsCache: statistics + attribute indexes for a collection of records (RecordsCache.scala:31-134).

Host-side mirror: value counts per attribute in one pass (RecordsCache.scala:75-96), one AttributeIndex per
matching attribute (:104-114), records transformed to integer value ids with -1 for missing (:117-133).
"""
import collections
import csv
from dataclasses import dataclass, field
from typing import List, Optional

import numpy as np

from .engine import SIMILARITY_FNS, AttributeIndex

# the AttributeIndex.build kind of each similarity function
_INDEX_KIND = {"ConstantSimilarityFn": "constant", "LevenshteinSimilarityFn": "levenshtein",
               "JaroWinklerSimilarityFn": "jaro-winkler"}


@dataclass
class SimilarityFn:
    """SimilarityFn.scala:50-107, plus JaroWinklerSimilarityFn: the Jaro-Winkler unit similarity of two strings
    (bytes, prefix scale 0.1) under the same threshold / maxSimilarity truncation as LevenshteinSimilarityFn."""
    name: str = "ConstantSimilarityFn"
    threshold: float = 7.0
    max_similarity: float = 10.0

    def __post_init__(self):
        if self.name not in SIMILARITY_FNS:
            raise ValueError(f"unsupported similarity function {self.name}")
        if self.name != "ConstantSimilarityFn":
            if not self.max_similarity > 0.0:
                raise ValueError("`maxSimilarity` must be positive")  # SimilarityFn.scala:59
            if not (0.0 <= self.threshold < self.max_similarity):
                raise ValueError("`threshold` must be in the interval [0, maxSimilarity)")  # :60-61

    @property
    def is_constant(self):
        return self.name == "ConstantSimilarityFn"

    @property
    def index_kind(self):
        """the `similarity` argument of AttributeIndex.build"""
        return _INDEX_KIND[self.name]


@dataclass
class Attribute:
    """package.scala:122-133 + BetaShapeParameters :164-168."""
    name: str
    similarity_fn: SimilarityFn = field(default_factory=SimilarityFn)
    alpha: float = 1.0
    beta: float = 1.0

    def __post_init__(self):
        if not (self.alpha > 0 and self.beta > 0):
            raise ValueError("shape parameters must be positive")

    @property
    def is_constant(self):
        return self.similarity_fn.is_constant


class RecordsCache:
    def __init__(self, attributes: List[Attribute], indexes: List[AttributeIndex], file_ids: List[str],
                 file_sizes: List[int], missing_counts=None):
        self.attributes = attributes
        self.indexes = indexes
        self.file_ids = file_ids          # sorted file id strings; position = integer file id
        self.file_sizes = file_sizes
        self.missing_counts = missing_counts

    @property
    def num_attributes(self):
        return len(self.attributes)

    @property
    def num_records(self):
        return int(sum(self.file_sizes))

    @classmethod
    def build(cls, values: List[List[Optional[str]]], file_of_record: List[str], attributes: List[Attribute],
              expected_max_cluster_size: int = 10):
        """RecordsCache.apply (RecordsCache.scala:68-115).  values[r][a] is a string or None (missing)."""
        if len(values) == 0:
            raise ValueError("no records")
        if len(values[0]) != len(attributes):
            raise ValueError("attribute specifications do not match the records")  # :72
        counts = [collections.Counter() for _ in attributes]
        fsz = collections.Counter()
        missing = collections.Counter()
        for rec, f in zip(values, file_of_record):
            fsz[f] += 1
            for a, v in enumerate(rec):
                if v is not None:
                    counts[a][v] += 1
                else:
                    missing[(f, a)] += 1
        indexes = []
        for a, attr in enumerate(attributes):
            vw = {k: float(v) for k, v in counts[a].items()}
            sf = attr.similarity_fn
            indexes.append(AttributeIndex.build(vw, sf.index_kind, sf.threshold, sf.max_similarity,
                                                expected_max_cluster_size))
        fids = sorted(fsz.keys())
        return cls(attributes, indexes, fids, [fsz[f] for f in fids], dict(missing))

    def transform_records(self, values, file_of_record):
        """_transformRecords (RecordsCache.scala:117-133): -> (x int32[R, A], file int32[R])."""
        R, A = len(values), self.num_attributes
        x = np.full((R, A), -1, np.int32)
        for a in range(A):
            ix = self.indexes[a]
            cache = {}
            for r in range(R):
                v = values[r][a]
                if v is None:
                    continue
                i = cache.get(v)
                if i is None:
                    i = ix.value_idx_of(v)
                    cache[v] = i
                x[r, a] = i
        fmap = {f: i for i, f in enumerate(self.file_ids)}
        file = np.array([fmap[f] for f in file_of_record], np.int32)
        return x, file


def read_csv(path, rec_id_col, attribute_names, file_id_col=None, ent_id_col=None, null_value="NA"):
    """Project.scala:173-180 + State.scala:350-371: CSV with header -> record ids, file ids, string values."""
    import gzip

    rec_ids, files, values, ent_ids = [], [], [], []
    opener = (lambda: gzip.open(path, "rt", newline="")) if str(path).endswith(".gz") else (lambda: open(path, newline=""))
    with opener() as fh:
        rd = csv.DictReader(fh)
        for row in rd:
            rec_ids.append(row[rec_id_col])
            files.append(row[file_id_col] if file_id_col else "0")
            values.append([None if (row[a] == null_value or row[a] == "") else row[a] for a in attribute_names])
            if ent_id_col:
                ent_ids.append(row[ent_id_col])
    return rec_ids, files, values, (ent_ids if ent_id_col else None)


# ---- columnar path (pyarrow): the same results without a Python loop over records ------------------------
def read_csv_columns(path, rec_id_col, attribute_names, file_id_col=None, ent_id_col=None, null_value="NA"):
    """read_csv through pyarrow.csv: -> (rec_ids, files, columns, ent_ids) with pyarrow string arrays (nulls =
    missing) instead of Python lists; .gz is handled by pyarrow.  Every column is read as a string, as the
    reference does (State.scala:350-371)."""
    import pyarrow as pa
    import pyarrow.compute as pc
    import pyarrow.csv as pacsv

    wanted = [rec_id_col] + list(attribute_names) + ([file_id_col] if file_id_col else []) + \
             ([ent_id_col] if ent_id_col else [])
    tbl = pacsv.read_csv(path, convert_options=pacsv.ConvertOptions(
        column_types={c: pa.string() for c in wanted}, include_columns=list(dict.fromkeys(wanted)),
        null_values=[], strings_can_be_null=False))

    def col(name):
        return tbl.column(name).combine_chunks()

    def nullable(a):  # the null marker and the empty string are missing values
        return pc.if_else(pc.or_(pc.equal(a, null_value), pc.equal(a, "")), pa.scalar(None, pa.string()), a)

    rec_ids = col(rec_id_col)
    files = col(file_id_col) if file_id_col else pa.array(["0"] * len(rec_ids), pa.string())
    columns = [nullable(col(a)) for a in attribute_names]
    return rec_ids, files, columns, (col(ent_id_col) if ent_id_col else None)


def build_cache_from_columns(columns, files, attributes: List[Attribute], expected_max_cluster_size: int = 10):
    """RecordsCache.build + transform_records on pyarrow string columns -> (cache, x int32[R, A], file int32[R])."""
    import pyarrow.compute as pc

    if len(columns) != len(attributes):
        raise ValueError("attribute specifications do not match the records")  # RecordsCache.scala:72
    R = len(files)
    if R == 0:
        raise ValueError("no records")
    fenc = files.dictionary_encode()
    fnames = fenc.dictionary.to_pylist()
    forder = np.argsort(np.asarray(fnames, dtype=object), kind="stable")  # sorted file ids; position = integer id
    frank = np.empty(len(fnames), np.int32)
    frank[forder] = np.arange(len(fnames), dtype=np.int32)
    fcodes = fenc.indices.to_numpy(zero_copy_only=False)
    file = frank[fcodes]
    fsz = np.bincount(file, minlength=len(fnames))
    x = np.full((R, len(attributes)), -1, np.int32)
    indexes, missing = [], {}
    for a, (colm, attr) in enumerate(zip(columns, attributes)):
        enc = colm.dictionary_encode()
        vals = enc.dictionary.to_pylist()
        codes = enc.indices.to_numpy(zero_copy_only=False)  # NaN / masked where null
        valid = np.asarray(pc.is_valid(colm).to_numpy(zero_copy_only=False), bool)
        ci = np.where(valid, np.nan_to_num(codes, nan=0).astype(np.int64), 0)
        cnt = np.bincount(ci[valid], minlength=len(vals))
        sf = attr.similarity_fn
        ix = AttributeIndex.build({v: float(c) for v, c in zip(vals, cnt) if c > 0}, sf.index_kind, sf.threshold,
                                  sf.max_similarity, expected_max_cluster_size)
        lut = np.array([ix.value_idx_of(v) if c > 0 else -1 for v, c in zip(vals, cnt)] + [-1], np.int32)
        x[:, a] = np.where(valid, lut[ci], -1)
        indexes.append(ix)
        miss = np.bincount(file[~valid], minlength=len(fnames))
        for f in np.flatnonzero(miss):
            missing[(fnames[forder[f]], a)] = int(miss[f])
    sorted_names = [fnames[i] for i in forder]
    cache = RecordsCache(attributes, indexes, sorted_names, [int(v) for v in fsz], missing)
    return cache, x, file
