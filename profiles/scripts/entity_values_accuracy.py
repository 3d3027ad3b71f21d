"""How often the posterior mode of an entity's value is its true value, against a majority vote of the values its
records carry, on synthetic data whose true entity values are known (synth.generate_encoded's ent_values).

One chain (PCG-II, --burnin sweeps, then --samples samples every --thinning sweeps, saveEntityValues on) over
--records records with the bench's 10 attributes (4 constant, 6 Levenshtein; distortion --distortion, 1 % missing,
4 blocks).  The center is the sMPC; only its clusters whose records are exactly one true entity are scored.  Per
attribute: the share of those clusters whose posterior mode (entity-value counts over the samples, ties to the
smallest value id) is the entity's true value, and the share whose majority vote of the recorded values (missing
values left out, ties to the smallest value id; a cluster whose values are all missing has no vote) is; each split
into clusters of one record and of two or more.  Card name and power limit are read in the same run.

    python profiles/scripts/entity_values_accuracy.py [--records 20000] [--distortion 0.1] [--seed 3]
"""
import argparse
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np  # noqa: E402

import dblink_b200 as D  # noqa: E402
from dblink_b200 import analysis_arrays as aa, analysis_gpu as ag, sampler, synth  # noqa: E402
from smpc_time import card  # noqa: E402


def majority(labels, codes, C):
    """Per cluster the most frequent non-missing code (ties to the smallest), -1 when all are missing."""
    ok = codes >= 0
    lab, val = labels[ok], codes[ok].astype(np.int64)
    out = np.full(C, -1, np.int64)
    if not len(lab):
        return out
    keys, n = np.unique(lab * (int(val.max()) + 1) + val, return_counts=True)
    cl, v = keys // (int(val.max()) + 1), keys % (int(val.max()) + 1)
    by = np.lexsort((v, -n, cl))
    lead = by[np.r_[True, cl[by][1:] != cl[by][:-1]]]
    out[cl[lead]] = v[lead]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=20000)
    ap.add_argument("--distortion", type=float, default=0.1)
    ap.add_argument("--seed", type=int, default=3)
    ap.add_argument("--burnin", type=int, default=500)
    ap.add_argument("--samples", type=int, default=100)
    ap.add_argument("--thinning", type=int, default=5)
    args = ap.parse_args()
    print(f"card: {card()}")
    attrs = synth.config_attrs(4)
    enc = synth.generate_encoded(args.seed, args.records, attrs, dup=0.10, distortion=args.distortion, missing=0.01)
    indexes, x, file, F = synth.build_encoded(enc)
    R = len(x)
    eng = D.GibbsEngine(indexes, [a.alpha for a in enc["attributes"]], [a.beta for a in enc["attributes"]], None,
                        args.seed, F)
    eng.init_state(x, file)
    split = [i for i, a in enumerate(attrs) if a.kind == "levenshtein"][:2]
    part = D.KDTreePartitioner(2, split).fit(eng.download_state()["y"])
    eng.set_partitioner(part)
    names = [a.name for a in attrs]
    values = [[ix.value_of(v) for v in range(ix.num_values)] for ix in indexes]
    out = tempfile.mkdtemp()
    sampler.sample(eng, [str(r) for r in range(R)], names, args.samples, out, args.burnin, args.thinning,
                   sampler="PCG-II", entity_values=values)
    eng.close()

    import pyarrow as pa

    ch = aa.read_chain_arrays(os.path.join(out, "linkage-chain.parquet"))
    rec = np.array([int(r) for r in ch.record_ids.to_pylist()])  # chain record index -> generated record
    labels = aa.canonical_clusters(ag.shared_most_probable_clusters(ch))
    C = int(labels.max()) + 1
    samples = aa.read_entity_values([out], ch, names, [pa.array(v, pa.string()) for v in values])
    modes, _, S = ag.entity_value_modes(labels, samples, [len(v) for v in values])

    ent = enc["ent_ids"][rec]
    size = np.bincount(labels, minlength=C)
    ent_size = np.bincount(enc["ent_ids"])
    first = np.full(C, -1, np.int64)
    first[labels[::-1]] = ent[::-1]  # the entity of some record of each cluster
    pure = np.bincount(labels, weights=(ent == first[labels]), minlength=C) == size
    exact = pure & (ent_size[first] == size)
    print(f"R = {R}, true entities = {len(ent_size)}, samples = {S} (burn-in {args.burnin}, thinning "
          f"{args.thinning}), distortion {args.distortion}, sMPC clusters = {C}, equal to a true entity = "
          f"{int(exact.sum())} ({int((exact & (size == 1)).sum())} of one record)")
    print("attribute,clusters,modeCorrect,majorityCorrect,modeCorrect1,majorityCorrect1,modeCorrect2+,"
          "majorityCorrect2+")
    for a, sa in enumerate(attrs):
        lut = {v: i for i, v in enumerate(values[a])}
        truth = np.array([lut.get(enc["vocabs"][a][c], -1) for c in enc["ent_values"][first[exact], a]])
        mode_ok = modes[a][exact] == truth
        vote_ok = majority(labels, x[rec, a], C)[exact] == truth  # x in generated order, labels in chain order
        one = size[exact] == 1
        row = [sa.name, int(exact.sum())]
        for m in (np.ones_like(one), one, ~one):
            row += [f"{mode_ok[m].mean():.4f}", f"{vote_ok[m].mean():.4f}"]
        print(",".join(str(v) for v in row))


if __name__ == "__main__":
    main()
