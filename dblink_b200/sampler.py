"""Chain driver: Sampler.sample (Sampler.scala:51-124) over a GibbsEngine / ShardedGibbs."""
import os
import shutil

from .writers import (DISTORTION_CHAIN, DiagnosticsWriter, DistortionChainWriter, EntityValuesChainWriter,
                      LinkageChainWriter, cluster_layout, entity_values_arrow, linkage_structure_arrow)

SUPPORTED_SAMPLERS = ("PCG-I", "PCG-II", "Gibbs", "Gibbs-Sequential")  # ProjectStep.scala:35


def sample(engine, record_ids, attribute_names, sample_size, output_path, burnin_interval=0, thinning_interval=1,
           write_buffer_size=10, sampler="PCG-I", population_size=None, on_sample=None, entity_values=None,
           distortion_columns=None):
    """Generates `sample_size` posterior samples by successively applying the transition operator; writes
    linkage-chain.parquet and diagnostics.csv under output_path.  Returns the number of sweeps performed.
    on_sample(summary, parts) sees every recorded sample; parts = {partition id: pyarrow ListArray of clusters}
    (`.to_pylist()` gives the lists of record ids).

    An engine holding K > 1 chains (GibbsEngine.init_chains / upload_chains) writes chain k's linkage-chain.parquet
    and diagnostics.csv under output_path/chain-<k>/, from one download of every chain's links per recorded sample;
    on_sample then sees every chain's sample, chain-major.

    entity_values: None, or per matching attribute its value strings in value-id order.  Given, each chain directory
    also gets entity-values-chain.parquet (writers.EntityValuesChainWriter), the value of every cluster's entity at
    every recorded sample; y comes from download_state (one chain), download_chains (K > 1) or, on a sharded engine,
    its download_state of y, block and link (a collective; rank 0 writes).  Not given, a new (not continued) chain
    removes the entity-values-chain.parquet an earlier chain left in its directory: the linkage chain it described
    is replaced.

    distortion_columns: None, or the column names of theta[A][F] attribute-major (writers.distortion_columns).  Given,
    each chain directory also gets distortion-probabilities-chain.csv (writers.DistortionChainWriter), theta of every
    recorded sample from the summary the step reads anyway; not given, a new chain removes such a file left by an
    earlier chain, as for entity values."""
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
    lw = dw = ew = tw = ids = None
    if writer:
        lw, dw, ew, tw = [], [], [], []
        for d in dirs:
            os.makedirs(d, exist_ok=True)
            lw.append(LinkageChainWriter(os.path.join(d, "linkage-chain.parquet"), write_buffer_size, continue_chain))
            dw.append(DiagnosticsWriter(os.path.join(d, "diagnostics.csv"), attribute_names, continue_chain))
            ev_path = os.path.join(d, "entity-values-chain.parquet")
            if entity_values is not None:
                ew.append(EntityValuesChainWriter(ev_path, attribute_names, write_buffer_size, continue_chain,
                                                  lw[-1].file_no))
            elif not continue_chain and os.path.isdir(ev_path):
                # a new chain without entity values: the values of an earlier chain in this directory would describe
                # other linkage rows under the same iterations and file names, so they go with that chain
                shutil.rmtree(ev_path)
            th_path = os.path.join(d, DISTORTION_CHAIN)
            if distortion_columns is not None:
                tw.append(DistortionChainWriter(th_path, distortion_columns, continue_chain))
            elif not continue_chain and os.path.exists(th_path):
                os.remove(th_path)  # the distortion probabilities of the replaced chain

        import pyarrow as pa

        ids = pa.array([str(r) for r in record_ids], pa.string())
        values = None if entity_values is None else [
            v if isinstance(v, pa.Array) else pa.array(list(v), pa.string()) for v in entity_values]

    def record():
        y = [None] * K
        if K == 1 and entity_values is None:
            link, blk = engine.links()  # sharded: a collective, every rank takes part
            samples = [(link, blk, engine.summary())]
        elif K == 1:
            # sharded (it has a rank): a collective over the arrays named, every rank takes part
            st = (engine.download_state(keys=("y", "block", "link")) if hasattr(engine, "rank") else
                  engine.download_state())
            samples, y = [(st["link"], st["block"], engine.summary())], [st["y"]]
        else:
            st = engine.download_chains(links_only=entity_values is None)
            samples = [(st[k]["link"], st[k]["block"], engine.chain_summary(k)) for k in range(K)]
            if entity_values is not None:
                y = [st[k]["y"] for k in range(K)]
        if not writer:
            return
        for k, (link, blk, s) in enumerate(samples):
            # one cluster order for both files
            layout = cluster_layout(link, blk) if entity_values is not None else None
            parts = linkage_structure_arrow(link, blk, ids, layout)  # {partition id: ListArray of clusters}
            lw[k].append(s["iteration"], parts)
            if entity_values is not None:
                ew[k].append(s["iteration"], entity_values_arrow(link, blk, y[k], values, layout))
            dw[k].write_row(s, pop)
            if distortion_columns is not None:
                tw[k].write_row(s["iteration"], s["theta"])
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
        for w in lw + ew + dw + tw:
            w.close()
    return done
