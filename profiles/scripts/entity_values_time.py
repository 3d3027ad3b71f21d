"""Time of the entity-value counts of a point estimate's clusters on a 1 M-record, 100-sample chain with 10
attributes: the device path (analysis_gpu.entity_value_modes, one dbl_values handle per attribute, every sample's
values uploaded from the host) against numpy's (analysis_arrays.entity_value_modes, on the first --numpy-samples
samples, reported as measured and scaled to all samples).  Host clock around work that ends in a synchronise; the
device path is run --repeats times after one warm-up run.

The chain is synthetic and seeded, shaped as smpc_time.py's: R records, links to 3R/4 entities, each sample moving
30 % of the records; each entity carries V values per attribute (V from 10 to 100 000), 10 % of them redrawn per sample.
The center is the labelling of the first sample.  numpy's time per sample grows with its held table, so the scaled
figure is an estimate (a low one).

--sample-step instead times what saveEntityValues adds to the sample step, per recorded sample: sampler.sample with
thinning 1 and write buffer 10 over 2 and over 12 samples, with the option off and on, alternating (off, on) three
times after a warm-up; the cost per sample is (t(12) - t(2)) / 10, which leaves out the writers' set-up.  On the
bench's 1M-record configuration (bench.py --config 4: seed 2, 64 blocks, PCG-II, engine seed 2024) and on RLdata10000
(4 blocks on fname_c1 / lname_c1, as bench.py's small configurations).

    python profiles/scripts/entity_values_time.py [--records 1000000] [--samples 100] [--numpy-samples 5]
    python profiles/scripts/entity_values_time.py --sample-step [--records 1000000]
"""
import argparse
import os
import shutil
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np  # noqa: E402

from dblink_b200 import analysis_arrays as aa, analysis_gpu as ag, sampler  # noqa: E402
from smpc_time import card, links  # noqa: E402

VOCAB = [10, 100, 1000, 3000, 10000, 30000, 100000, 50, 500, 5000]


def value_samples(link_list, E, seed):
    rng = np.random.default_rng(seed)
    y = np.stack([rng.integers(0, V, E) for V in VOCAB]).astype(np.int32)  # [A][E]
    out = []
    for link in link_list:
        move = rng.random(y.shape) < 0.1
        y = np.where(move, np.stack([rng.integers(0, V, E) for V in VOCAB]).astype(np.int32), y)
        out.append(y[:, link])
    return out


def step_cost(eng, rec_ids, names, values, label, samp="PCG-II"):
    """Per recorded sample seconds of sampler.sample with entity values off and on: (t(12) - t(2)) / 10, three
    alternating rounds after a warm-up."""
    import torch

    tmp = tempfile.mkdtemp()
    try:
        def run(n, on):
            d = os.path.join(tmp, f"{'on' if on else 'off'}-{n}")
            torch.cuda.synchronize()
            t = time.perf_counter()
            sampler.sample(eng, rec_ids, names, n, d, 0, 1, 10, samp, entity_values=values if on else None)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t
            shutil.rmtree(d)
            return dt

        eng.sweep(samp, 5)
        run(2, False), run(2, True)  # warm-up
        per = {False: [], True: []}
        for _ in range(3):
            for on in (False, True):
                per[on].append((run(12, on) - run(2, on)) / 10)
        off_ms = [1e3 * x for x in per[False]]
        on_ms = [1e3 * x for x in per[True]]
        print(f"{label}: ms per recorded sample (one sweep + recording), off: "
              + ", ".join(f"{x:.1f}" for x in off_ms) + "; on: " + ", ".join(f"{x:.1f}" for x in on_ms)
              + f"; median added: {np.median(on_ms) - np.median(off_ms):.1f} ms")
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


def sample_step(args):
    import dblink_b200 as D
    from dblink_b200 import config, synth
    from dblink_b200.project import Project

    print(f"card: {card()}")
    attrs = synth.config_attrs(4)
    enc = synth.generate_encoded(2, args.records, attrs, dup=0.10, distortion=0.05, missing=0.01, n_files=2)
    indexes, x, file, F = synth.build_encoded(enc)
    eng = D.GibbsEngine(indexes, [a.alpha for a in enc["attributes"]], [a.beta for a in enc["attributes"]], None,
                        2024, F)
    eng.init_state(x, file)
    split = [i for i, a in enumerate(attrs) if a.kind == "levenshtein"][:6]
    part = D.KDTreePartitioner(6, split).fit(eng.download_state()["y"])
    eng.set_partitioner(part)
    values = [[ix.value_of(v) for v in range(ix.num_values)] for ix in indexes]
    step_cost(eng, [str(r) for r in range(len(x))], [a.name for a in attrs], values,
              f"synthetic {len(x)} records / 10 attrs / 64 blocks, PCG-II")
    eng.close()

    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_host_pipeline import GOLDEN, make_conf

    conf = make_conf(os.path.join(GOLDEN, "RLdata10000.csv.gz"), tempfile.mkdtemp() + "/", 2,
                     '["fname_c1", "lname_c1"]')
    conf = conf.replace("lowDistortion : {alpha : 0.5, beta : 50.0}", "lowDistortion : {alpha : 10.0, beta : 1000.0}")
    p = Project(config.parse_string(conf), base_dir="")
    eng = p.generate_initial_state()
    step_cost(eng, p.load()["rec_ids"], [a.name for a in p.matching_attributes], p.attribute_values(),
              "RLdata10000 / 4 blocks, PCG-II")
    eng.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=1_000_000)
    ap.add_argument("--samples", type=int, default=100)
    ap.add_argument("--numpy-samples", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--sample-step", action="store_true")
    args = ap.parse_args()
    if args.sample_step:
        return sample_step(args)
    R, S = args.records, args.samples
    ls, _ = links(R, S, seed=1)
    vals = value_samples(ls, (3 * R) // 4, seed=2)
    labels = aa.canonical_clusters(ls[0])
    print(f"card: {card()}")
    print(f"R = {R}, S = {S}, A = {len(VOCAB)}, clusters = {int(labels.max()) + 1}, values = {VOCAB}")
    times = []
    for i in range(args.repeats + 1):
        t = time.perf_counter()
        m_gpu, c_gpu, _ = ag.entity_value_modes(labels, iter(vals), VOCAB)
        times.append(time.perf_counter() - t)
    print("device (s, after one warm-up): " + ", ".join(f"{x:.3f}" for x in times[1:]))
    n = args.numpy_samples
    t = time.perf_counter()
    m_np, c_np, _ = aa.entity_value_modes(labels, iter(vals[:n]), VOCAB)
    t_np = time.perf_counter() - t
    m_sub, c_sub, _ = ag.entity_value_modes(labels, iter(vals[:n]), VOCAB)
    assert np.array_equal(m_np, m_sub) and np.array_equal(c_np, c_sub)
    print(f"numpy (s): {t_np:.2f} on {n} samples, {t_np * S / n:.1f} scaled linearly to {S} (an estimate: the held "
          f"table grows); device equal on those {n}")


if __name__ == "__main__":
    main()
