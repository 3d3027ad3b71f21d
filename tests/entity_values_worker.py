"""Worker of test_gpu_entity_values: `python -m torch.distributed.run ... tests/entity_values_worker.py`, one rank per
GPU over NCCL.  Sampler.sample over ShardedGibbs twice from the same seed, with and without entity values: the
linkage chains must be equal; rank 0's entity-values chain must hold, for the last sample, the entity values of the
final state gathered from every rank, and rank 0's two chain files must hold, sample by sample, what a one-GPU
GibbsEngine run from the same seed and the same k-d tree writes."""
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    import torch
    import torch.distributed as dist

    import dblink_b200 as D
    from dblink_b200 import analysis_arrays as aa, sampler
    from dblink_b200.distributed import ShardedGibbs
    from helpers import synth_problem

    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    rank = dist.get_rank()
    g = synth_problem(seed=6, R=900, n_files=2)
    rc = D.RecordsCache.build(g["values"], g["files"], g["attributes"])
    x, file = rc.transform_records(g["values"], g["files"])
    names = [a.name for a in g["attributes"]]
    values = [[ix.value_of(v) for v in range(ix.num_values)] for ix in rc.indexes]
    ids = [f"r{i}" for i in range(len(x))]
    out = [tempfile.mkdtemp() if rank == 0 else None]
    dist.broadcast_object_list(out, src=0)
    dirs = [os.path.join(out[0], "on"), os.path.join(out[0], "off")]
    final = None
    for d, ev in zip(dirs, (values, None)):
        eng = ShardedGibbs(rc.indexes, [a.alpha for a in g["attributes"]], [a.beta for a in g["attributes"]], seed=3,
                           num_files=len(rc.file_ids), levels=2, split_attrs=(2, 3))
        eng.init_state(x, file)
        sampler.sample(eng, ids, names, 4, d, burnin_interval=2, thinning_interval=3, write_buffer_size=3,
                       sampler="PCG-I", entity_values=ev)
        if ev is not None:
            final = eng.download_state(keys=("y", "link"))  # a collective: every rank takes part
    dist.barrier()
    if rank == 0:
        import pyarrow as pa

        # the same chain on one GPU: one engine, the k-d tree fitted as ShardedGibbs.init_state fits it
        one = os.path.join(out[0], "one")
        eng = D.GibbsEngine(rc.indexes, [a.alpha for a in g["attributes"]], [a.beta for a in g["attributes"]], None, 3,
                            len(rc.file_ids))
        eng.init_state(x, file)
        part = D.KDTreePartitioner(2, (2, 3)).fit(eng.download_state()["y"])
        eng.set_partitioner(part)
        sampler.sample(eng, ids, names, 4, one, burnin_interval=2, thinning_interval=3, write_buffer_size=3,
                       sampler="PCG-I", entity_values=values)
        eng.close()

        strings = [pa.array(v, pa.string()) for v in values]
        on, off, single = (aa.read_chain_arrays(os.path.join(d, "linkage-chain.parquet")) for d in dirs + [one])
        assert on.iterations.tolist() == off.iterations.tolist() == single.iterations.tolist() == [2, 5, 8, 11]
        assert on.record_ids.equals(single.record_ids)
        for other in (off, single):
            assert all(np.array_equal(a[i], b[i]) for a, b in zip(on.samples, other.samples) for i in range(3))
        got = list(aa.read_entity_values([dirs[0]], on, names, strings))
        want_one = list(aa.read_entity_values([one], single, names, strings))
        assert len(got) == len(want_one) == 4
        assert all(np.array_equal(a, b) for a, b in zip(got, want_one))  # every sample, not only the last
        pos = {r: i for i, r in enumerate(on.record_ids.to_pylist())}
        want = np.empty_like(got[-1])
        want[:, np.array([pos[r] for r in ids])] = final["y"][final["link"]].T
        assert np.array_equal(got[-1], want)
        print(f"sharded entity values ok on {dist.get_world_size()} ranks")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
