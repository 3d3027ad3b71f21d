"""Attribute-index build time, GPU kernels vs host loops (all host threads), for a vocabulary of V strings.

    index_time.py [V] [gpu] [levenshtein | jaro-winkler]

`gpu` skips the host build; the similarity defaults to levenshtein at threshold 7/10 (jaro-winkler: 8.5/10)."""
import os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import numpy as np
import dblink_b200 as D
from dblink_b200 import synth
THRESHOLDS = {"levenshtein": 7.0, "jaro-winkler": 8.5}
args = [a for a in sys.argv[1:] if a not in THRESHOLDS]
sim = next((a for a in sys.argv[1:] if a in THRESHOLDS), "levenshtein")
thr = THRESHOLDS[sim]
V = int(args[0]) if args else 50000
host_too = len(args) <= 1 or args[1] != "gpu"
rng = np.random.default_rng(7)
strings, _ = synth._string_vocab(rng, V)
strings = list(dict.fromkeys(strings))
vw = {s: float(1 + (i * 7919) % 13) for i, s in enumerate(strings)}
print("V =", len(vw), "mean length", np.mean([len(s) for s in strings]), "similarity", sim, thr, "/ 10")
os.environ["DBL_INDEX_GPU"] = "1"
D.AttributeIndex.build(dict(list(vw.items())[:3000]), sim, thr, 10.0)  # warm-up (context, module load)
t = time.time(); g = D.AttributeIndex.build(vw, sim, thr, 10.0); tg = time.time() - t
print(f"GPU build: {tg:.2f} s, nnz {g.nnz}, hash slots {g.hash_slots}")
if host_too:
    os.environ["DBL_INDEX_GPU"] = "0"
    t = time.time(); h = D.AttributeIndex.build(vw, sim, thr, 10.0); th = time.time() - t
    print(f"host build ({len(os.sched_getaffinity(0))} cpus visible): {th:.2f} s, nnz {h.nnz}; speed-up {th / tg:.1f}x")
    a, b = g.tables(), h.tables()
    print("identical tables:", all(np.array_equal(a[k], b[k]) for k in a))
