"""Chain driver: Sampler.sample (Sampler.scala:51-124) over a GibbsEngine / ShardedGibbs."""
import os

from .writers import DiagnosticsWriter, LinkageChainWriter, linkage_structure_arrow

SUPPORTED_SAMPLERS = ("PCG-I", "PCG-II", "Gibbs", "Gibbs-Sequential")  # ProjectStep.scala:35


def sample(engine, record_ids, attribute_names, sample_size, output_path, burnin_interval=0, thinning_interval=1,
           write_buffer_size=10, sampler="PCG-I", population_size=None, on_sample=None):
    """Generates `sample_size` posterior samples by successively applying the transition operator; writes
    linkage-chain.parquet and diagnostics.csv under output_path.  Returns the number of sweeps performed.
    on_sample(summary, parts) sees every recorded sample; parts = {partition id: pyarrow ListArray of clusters}
    (`.to_pylist()` gives the lists of record ids).

    An engine holding K > 1 chains (GibbsEngine.init_chains / upload_chains) writes chain k's linkage-chain.parquet
    and diagnostics.csv under output_path/chain-<k>/, from one download of every chain's links per recorded sample;
    on_sample then sees every chain's sample, chain-major."""
    if sample_size <= 0:
        raise ValueError("`sampleSize` must be positive.")            # Sampler.scala:61
    if burnin_interval < 0:
        raise ValueError("`burninInterval` must be non-negative.")    # :62
    if thinning_interval <= 0:
        raise ValueError("`thinningInterval` must be positive.")      # :63
    if write_buffer_size <= 0:
        raise ValueError("`writeBufferSize` must be positive.")       # :65
    if sampler not in SUPPORTED_SAMPLERS:
        raise ValueError(f"sampler must be one of {', '.join(SUPPORTED_SAMPLERS)}.")  # ProjectStep.scala:44
    writer = getattr(engine, "rank", 0) == 0  # a sharded engine runs on every rank; rank 0 writes the outputs
    if writer:
        os.makedirs(output_path, exist_ok=True)
    initial_iteration = engine.iteration
    continue_chain = initial_iteration != 0
    pop = population_size if population_size is not None else engine.num_entities
    K = getattr(engine, "num_chains", 1)
    dirs = [output_path] if K == 1 else [os.path.join(output_path, f"chain-{k}") for k in range(K)]
    lw = dw = ids = None
    if writer:
        lw, dw = [], []
        for d in dirs:
            os.makedirs(d, exist_ok=True)
            lw.append(LinkageChainWriter(os.path.join(d, "linkage-chain.parquet"), write_buffer_size, continue_chain))
            dw.append(DiagnosticsWriter(os.path.join(d, "diagnostics.csv"), attribute_names, continue_chain))

        import pyarrow as pa

        ids = pa.array([str(r) for r in record_ids], pa.string())

    def record():
        if K == 1:
            link, blk = engine.links()  # sharded: a collective, every rank takes part
            samples = [(link, blk, engine.summary())]
        else:
            st = engine.download_chains(links_only=True)
            samples = [(st[k]["link"], st[k]["block"], engine.chain_summary(k)) for k in range(K)]
        if not writer:
            return
        for k, (link, blk, s) in enumerate(samples):
            parts = linkage_structure_arrow(link, blk, ids)  # {partition id: ListArray of clusters}
            lw[k].append(s["iteration"], parts)
            dw[k].write_row(s, pop)
            if on_sample:
                on_sample(s, parts)

    if not continue_chain and burnin_interval == 0:
        record()  # the initial state is a sample (Sampler.scala:84-89)
    count, done = 0, 0
    while count < sample_size:
        # all the sweeps up to the next recorded iteration in ONE call: they are enqueued back to back on the device
        # and the host waits once (Sampler.scala:92-115 applies nextState one at a time)
        completed = engine.iteration - initial_iteration
        if completed < burnin_interval:
            step = burnin_interval - completed
        else:
            step = thinning_interval - (completed - burnin_interval) % thinning_interval
        engine.sweep(sampler, step)
        done += step
        record()
        count += 1
    if writer:
        for w in lw + dw:
            w.close()
    return done
