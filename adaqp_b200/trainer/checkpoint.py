"""Checkpoints of a training run: save, resume bit for bit, and load trained weights for prediction (DESIGN §12).

    <checkpoint_dir>/epoch{E:05d}/model.pt       model + Adam state_dict (identical on every rank; rank 0 writes it)
                                  rank{r}.pt     per-rank RNG states, Assigner state, Recorder rows 1..E, records
                                  manifest.json  format version, epoch, run fields, per-rank partition digests
    <checkpoint_dir>/latest                      name of the newest complete epoch directory
    <checkpoint_dir>/best/model.pt, manifest.json  the epoch with the best validation metric (model only)

A checkpoint is written under `.tmp-<name>` and renamed by rank 0 after a barrier, so a run killed mid-write
leaves no directory that looks valid.  Every file is read back with `torch.load(..., weights_only=True)`.
"""
from __future__ import annotations

import hashlib
import json
import os
import shutil
from typing import Dict, List, Optional

import numpy as np
import torch

from ..assigner import Assigner as assigner
from ..communicator import Communicator as comm
from ..communicator.p2p import layer_key_dims, quantisable
from ..helper import BitType
from ..manager import GraphEngine as engine
from ..model.registry import MODELS

FORMAT_VERSION = 1
# what a resumed run must share with the run that wrote the checkpoint; the first five also fix the weights' shapes
RUN_FIELDS = ("dataset", "model_name", "aggregator_type", "gat_heads", "layer_dims", "num_parts", "mode",
              "assign_scheme", "key_dims")
MODEL_FIELDS = RUN_FIELDS[:5]
# fields added after format 1 was fixed, compared on resume and on prediction: a manifest written before a field
# existed reads as null, which is what runs of the models without it record.  `propagation` is APPNP's {k, alpha}
# and GCNII's {layers, alpha, theta}.
ADDED_FIELDS = ("propagation",)


# ----------------------------------------------------------------------------- descriptions of the run
def run_fields(config: dict, key_dims: Optional[Dict[str, int]]) -> dict:
    """The manifest's description of a run, from the Trainer's resolved config and its exchange key widths
    (None: the reference's keys, as the Assigner builds them)."""
    data, model, rt = config["data"], config["model"], config["runtime"]
    L, H = int(model["num_layers"]), int(model["hidden_dim"])
    layer_dims = [int(data["num_feats"])] + [H] * (L - 1) + [int(data["num_classes"])]
    if key_dims is None:
        key_dims = {k: v for k, v in layer_key_dims(layer_dims[:-1]).items() if quantisable(k)}
    return {"dataset": rt["dataset"], "model_name": rt["model_name"], "aggregator_type": model["aggregator_type"],
            "gat_heads": int(model["gat_heads"]), "layer_dims": layer_dims,
            "num_parts": int(rt["num_parts"]), "mode": rt["mode"], "assign_scheme": rt["assign_scheme"],
            "key_dims": {k: int(v) for k, v in key_dims.items()},
            "propagation": MODELS[rt["model_name"]].propagation(config)}


def partition_digest(layout) -> dict:
    """Enough of a rank's partition to tell that a resumed run reads the same one."""
    h = hashlib.sha256()
    for a in (layout.indptr, layout.indices):
        a = np.ascontiguousarray(a)
        h.update(str(a.dtype).encode())
        h.update(a.tobytes())
    return {"n_inner": int(layout.n_inner), "n_halo": int(layout.n_halo),
            "send_idx": {str(p): [int(lo), int(hi)] for p, (lo, hi) in sorted(layout.send_idx.items())},
            "csr_sha256": h.hexdigest()}


def resolve(path: str, checkpoint_dir: Optional[str]) -> str:
    """`auto` names `<checkpoint_dir>/latest`; anything else is a checkpoint directory."""
    if path != "auto":
        return path
    if not checkpoint_dir:
        raise ValueError("resume='auto' needs checkpoint_dir")
    latest = os.path.join(checkpoint_dir, "latest")
    if not os.path.exists(latest):
        raise FileNotFoundError(f"no checkpoint to resume: {latest} does not exist")
    with open(latest) as f:
        return os.path.join(checkpoint_dir, f.read().strip())


def read_manifest(path: str) -> dict:
    m = os.path.join(path, "manifest.json")
    if not os.path.exists(m):
        raise FileNotFoundError(f"{path} is not a checkpoint: {m} does not exist")
    with open(m) as f:
        return json.load(f)


def _compare(manifest: dict, fields: dict, names) -> Optional[ValueError]:
    if manifest.get("format") != FORMAT_VERSION:
        return ValueError(f"checkpoint format {manifest.get('format')} is not {FORMAT_VERSION}")
    for k in names:
        if manifest["run"].get(k) != fields[k]:
            return ValueError(f"checkpoint field {k!r} is {manifest['run'].get(k)!r}, this run has {fields[k]!r}")
    return None


def resume_error(path: str, fields: dict, digest: dict, rank: int, num_epoches: int) -> Optional[Exception]:
    """Why this rank cannot resume from `path` (None: it can).  Checked before any device work: every manifest
    field against this run, every rank's file, this rank's partition digest, and that epochs are left to run."""
    try:
        manifest = read_manifest(path)
    except FileNotFoundError as e:
        return e
    err = _compare(manifest, fields, RUN_FIELDS + ADDED_FIELDS)
    if err is not None:
        return err
    for r in range(fields["num_parts"]):
        if not os.path.exists(os.path.join(path, f"rank{r}.pt")):
            return FileNotFoundError(f"checkpoint {path} has no rank{r}.pt")
    if not os.path.exists(os.path.join(path, "model.pt")):
        return FileNotFoundError(f"checkpoint {path} has no model.pt")
    saved = manifest["partitions"][rank]
    for k in ("n_inner", "n_halo", "send_idx", "csr_sha256"):
        if saved[k] != digest[k]:
            return ValueError(f"checkpoint field 'partitions[{rank}].{k}' does not match this run's partition")
    if manifest["epoch"] >= num_epoches:
        return ValueError(f"checkpoint epoch {manifest['epoch']} >= num_epoches {num_epoches}: nothing left to train")
    return None


def check_resume(path: str, fields: dict, digest: dict, num_epoches: int) -> int:
    """Collective: every rank raises the same error when any rank cannot resume.  Returns the checkpoint's epoch."""
    err = resume_error(path, fields, digest, comm.get_rank(), num_epoches)
    errs = comm.gather_all(None if err is None else (type(err).__name__, str(err)))
    first = next((e for e in errs if e is not None), None)
    if first is not None:
        kind = {"ValueError": ValueError, "FileNotFoundError": FileNotFoundError}.get(first[0], RuntimeError)
        raise kind(first[1])
    return int(read_manifest(path)["epoch"])


# ----------------------------------------------------------------------------- tensors in, tensors out
def _cpu(obj):
    if isinstance(obj, torch.Tensor):
        return obj.detach().cpu().clone()
    if isinstance(obj, dict):
        return {k: _cpu(v) for k, v in obj.items()}
    if isinstance(obj, (list, tuple)):
        return type(obj)(_cpu(v) for v in obj)
    return obj


def _digest(obj, h) -> None:
    if isinstance(obj, torch.Tensor):
        h.update(f"T{obj.dtype}{tuple(obj.shape)}".encode())
        h.update(obj.reshape(-1).contiguous().view(torch.uint8).numpy().tobytes())
    elif isinstance(obj, dict):
        for k in sorted(obj, key=str):
            h.update(f"K{k!r}".encode())
            _digest(obj[k], h)
    elif isinstance(obj, (list, tuple)):
        h.update(f"L{len(obj)}".encode())
        for v in obj:
            _digest(v, h)
    else:
        h.update(f"V{obj!r}".encode())


def sha256_of(obj) -> str:
    h = hashlib.sha256()
    _digest(obj, h)
    return h.hexdigest()


def _np_rng_state() -> dict:
    name, keys, pos, has_gauss, cached = np.random.get_state()
    return {"name": name, "keys": torch.from_numpy(keys.astype(np.int64)), "pos": int(pos),
            "has_gauss": int(has_gauss), "cached_gaussian": float(cached)}


def _set_np_rng_state(s: dict):
    np.random.set_state((s["name"], s["keys"].numpy().astype(np.uint32), s["pos"], s["has_gauss"], s["cached_gaussian"]))


def _load(path: str):
    return torch.load(path, map_location="cpu", weights_only=True)


def _write_json(path: str, obj):
    with open(path, "w") as f:
        json.dump(obj, f, indent=1)


# ----------------------------------------------------------------------------- save
def save(root: str, epoch: int, model, optimizer, fields: dict, digest: dict, records: Dict[str, list]) -> str:
    """Collective: write `<root>/epoch{epoch:05d}` and point `<root>/latest` at it."""
    rank, W = comm.get_rank(), comm.get_world_size()
    name = f"epoch{epoch:05d}"
    tmp, final = os.path.join(root, f".tmp-{name}"), os.path.join(root, name)
    if comm.ctx.device.type == "cuda":
        torch.cuda.synchronize(comm.ctx.device)            # the traced accumulators are written on a side stream
    if rank == 0:
        shutil.rmtree(tmp, ignore_errors=True)
        os.makedirs(tmp)
    comm.barrier()
    state = {"model": _cpu(model.state_dict()), "optimizer": _cpu(optimizer.state_dict())}
    sha = sha256_of(state)
    shas = comm.gather_all(sha)
    if any(s != shas[0] for s in shas):               # raised on every rank, so that none waits in a barrier
        raise RuntimeError(f"the ranks' model / optimizer states differ ({shas}): the ranks have diverged")
    dev = comm.ctx.device
    rank_state = {"epoch": int(epoch),
                  "rng": {"torch": torch.get_rng_state(),
                          "cuda": torch.cuda.get_rng_state(dev) if dev.type == "cuda" else None,
                          "numpy": _np_rng_state()},
                  "assigner": assigner.ctx.state_dict(),
                  "recorder": engine.ctx.recorder.epoches_metrics[:epoch].clone(),
                  "records": {k: torch.tensor(v, dtype=torch.float64) for k, v in records.items()}}
    torch.save(rank_state, os.path.join(tmp, f"rank{rank}.pt"))
    digests = comm.gather_all(digest)
    if rank == 0:
        torch.save(state, os.path.join(tmp, "model.pt"))
        _write_json(os.path.join(tmp, "manifest.json"), {"format": FORMAT_VERSION, "epoch": int(epoch), "run": fields,
                                                         "partitions": digests, "model_sha256": sha})
    comm.barrier()                                         # every rank's file is complete
    if rank == 0:
        if os.path.exists(final):
            shutil.rmtree(final)
        os.replace(tmp, final)
        with open(os.path.join(root, ".latest.tmp"), "w") as f:
            f.write(name + "\n")
        os.replace(os.path.join(root, ".latest.tmp"), os.path.join(root, "latest"))
    comm.barrier()
    return final


def save_best(root: str, epoch: int, model, fields: dict, metrics: List[float], metric_name: str):
    """Rank 0 only: `<root>/best` = this epoch's model and metrics (replaced whole, never half-written)."""
    tmp, old, best = (os.path.join(root, n) for n in (".tmp-best", ".old-best", "best"))
    shutil.rmtree(tmp, ignore_errors=True)
    os.makedirs(tmp)
    state = {"model": _cpu(model.state_dict())}
    torch.save(state, os.path.join(tmp, "model.pt"))
    _write_json(os.path.join(tmp, "manifest.json"),
                {"format": FORMAT_VERSION, "epoch": int(epoch), "run": fields, "metric": metric_name,
                 "train": float(metrics[0]), "val": float(metrics[1]), "test": float(metrics[2]),
                 "model_sha256": sha256_of(state)})
    shutil.rmtree(old, ignore_errors=True)
    if os.path.exists(best):
        os.replace(best, old)
    os.replace(tmp, best)
    shutil.rmtree(old, ignore_errors=True)


# ----------------------------------------------------------------------------- load
def load_run(path: str, model, optimizer) -> dict:
    """Restore model, optimizer, Assigner, Recorder rows and RNG states from `path` (already checked by
    check_resume); re-apply the saved bit assignment.  Returns the rank's records."""
    rank = comm.get_rank()
    state = _load(os.path.join(path, "model.pt"))
    mine = _load(os.path.join(path, f"rank{rank}.pt"))
    model.load_state_dict(state["model"])
    optimizer.load_state_dict(state["optimizer"])
    asg, eng = assigner.ctx, engine.ctx
    asg.load_state_dict(mine["assigner"])
    if eng.bit_type == BitType.QUANT and asg.assignment is not None:
        # the Trainer drew a fresh first assignment while it was built: the saved one replaces it
        comm.ctx.update_buffer(asg.assignment)
    E = int(mine["epoch"])
    eng.recorder.epoches_metrics[:E] = mine["recorder"]
    torch.set_rng_state(mine["rng"]["torch"])
    if mine["rng"]["cuda"] is not None:
        torch.cuda.set_rng_state(mine["rng"]["cuda"], comm.ctx.device)
        torch.cuda.synchronize(comm.ctx.device)
    _set_np_rng_state(mine["rng"]["numpy"])
    return {k: v.tolist() for k, v in mine["records"].items()}


def load_weights(path: str, model, fields: dict) -> dict:
    """Model weights only (epoch or best checkpoint), for prediction: the model fields must match; the partition,
    `num_parts` and `mode` may differ, since weights do not depend on them.  Returns the manifest."""
    manifest = read_manifest(path)
    err = _compare(manifest, fields, MODEL_FIELDS + ADDED_FIELDS)
    if err is not None:
        raise err
    model.load_state_dict(_load(os.path.join(path, "model.pt"))["model"])
    return manifest
