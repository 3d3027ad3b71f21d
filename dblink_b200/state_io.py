"""Save / resume of the chain state (State.save / State.read, State.scala:122-193).

The reference writes a JVM-serialised `driver-state` plus `partitions-state.parquet`; neither can be produced or
read without a JVM, so this build keeps the same *content* in one portable file, `state.npz`, under the output
path: iteration, theta, z, links, entity values, population size, seed, and a fingerprint of the model tables so a
state is never resumed against different data or attribute specifications.
"""
import hashlib
import os

import numpy as np

STATE_FILE = "state.npz"


def model_fingerprint(indexes, x, file_ids, alpha, beta, extra=()):
    """Everything a saved state depends on: the tables, the encoded records, the priors and `extra` (random seed,
    population size, partitioner levels / attributes -- they fix the Philox key, E and the partition function)."""
    h = hashlib.sha256()
    for ix in indexes:
        t = ix.tables()
        for k in ("phi", "norm", "rowptr", "col", "expsim"):
            h.update(np.ascontiguousarray(t[k]).tobytes())
    h.update(np.ascontiguousarray(x).tobytes())
    h.update(np.ascontiguousarray(file_ids).tobytes())
    h.update(np.asarray(alpha, np.float64).tobytes())
    h.update(np.asarray(beta, np.float64).tobytes())
    h.update(repr(tuple(extra)).encode())
    return h.hexdigest()


def save_state(engine, output_path, fingerprint, seed):
    st = engine.download_state()
    os.makedirs(output_path, exist_ok=True)
    tmp = os.path.join(output_path, STATE_FILE + ".tmp.npz")
    np.savez_compressed(tmp, iteration=np.int64(engine.iteration), theta=st["theta"], z=np.packbits(st["z"], axis=1),
                        n_attrs=np.int64(st["z"].shape[1]), link=st["link"], y=st["y"],
                        population_size=np.int64(engine.num_entities), seed=np.int64(seed),
                        fingerprint=np.array(fingerprint))
    os.replace(tmp, os.path.join(output_path, STATE_FILE))


def save_chain_states(engine, output_paths, fingerprint, seeds):
    """The K chains of a batched engine, chain k's state.npz under output_paths[k] (same format as save_state)."""
    for path, st, seed in zip(output_paths, engine.download_chains(), seeds):
        os.makedirs(path, exist_ok=True)
        tmp = os.path.join(path, STATE_FILE + ".tmp.npz")
        np.savez_compressed(tmp, iteration=np.int64(engine.iteration), theta=st["theta"],
                            z=np.packbits(st["z"], axis=1), n_attrs=np.int64(st["z"].shape[1]), link=st["link"],
                            y=st["y"], population_size=np.int64(engine.num_entities), seed=np.int64(seed),
                            fingerprint=np.array(fingerprint))
        os.replace(tmp, os.path.join(path, STATE_FILE))


def saved_state_exists(output_path):
    return os.path.exists(os.path.join(output_path, STATE_FILE))


def load_state(output_path, fingerprint=None):
    d = np.load(os.path.join(output_path, STATE_FILE), allow_pickle=False)
    if fingerprint is not None and str(d["fingerprint"]) != fingerprint:
        raise ValueError("saved state does not match the data / attribute specifications of this project")
    A = int(d["n_attrs"])
    z = np.unpackbits(d["z"], axis=1)[:, :A]
    return {"iteration": int(d["iteration"]), "theta": d["theta"], "z": z, "link": d["link"], "y": d["y"],
            "population_size": int(d["population_size"]), "seed": int(d["seed"])}
