"""Table / optimizer-slot checkpoint I/O (SURVEY 8f N4).  The reference's tf2 path has none (``save_interval`` is
assigned and never used, tf2_examples/bpr_citeulike.py:16); 51 GB sharded tables need one to be practical.
Format: one ``.npz`` with ``var/<k>`` in ``model.variables`` order and their ``names``, plus ``slot<j>/<k>`` and
``iterations`` when an optimizer is given.  Row-sharded models: ``HomeRoutedPairwise.save_shard / load_shard``
(openrec_b200/sharded.py), one file per rank.

A Keras model creates its Dense layers during the first call, so an un-called DLRM / GMF does not have all of its
variables yet: saving or loading such a model would silently drop the MLP weights.  Both directions therefore insist
that the variable lists match (count, names, shapes); ``load(..., build=fn)`` lets the caller run one forward call
(``fn()``) first when the model is fresh.

A bfloat16 table (``embedding_dtype="bfloat16"``) is saved as its raw 16-bit words (uint16) with ``dtype/<k>`` =
"bfloat16", so a round trip is bit-exact; loading it into a float32 variable, or a float32 one into a bfloat16 variable,
is refused."""
from __future__ import annotations

import numpy as np
import torch


def _unbuilt(model):
    """Names of sub-layers that have not created their variables yet (keras `built` flag)."""
    out = []
    for name, sub in vars(model).items():
        for layer in getattr(sub, "layers", [sub]):
            if hasattr(layer, "built") and not layer.built:
                out.append(f"{name}.{type(layer).__name__}")
    return out


def _dtype(v):
    return "bfloat16" if v.t.dtype == torch.bfloat16 else "float32"


def _words(v):
    """the raw bf16 bits of a bfloat16 variable, as uint16"""
    return v.t.detach().view(torch.int16).cpu().numpy().view(np.uint16)


def save(path, model, optimizer=None):
    pending = _unbuilt(model)
    if pending:
        raise ValueError(f"checkpoint.save: {pending} have no variables yet (call the model once first); a checkpoint "
                         "written now would silently lack them")
    variables = model.variables
    out = {f"var/{k}": _words(v) if _dtype(v) == "bfloat16" else v.numpy() for k, v in enumerate(variables)}
    out.update({f"dtype/{k}": np.array("bfloat16") for k, v in enumerate(variables) if _dtype(v) == "bfloat16"})
    out["names"] = np.array([v.name for v in variables])
    if optimizer is not None:
        out["iterations"] = np.int64(optimizer.iterations)
        for k, v in enumerate(variables):
            for j, s in enumerate(optimizer.slots_if_any(v)):
                if s is not None:
                    out[f"slot{j}/{k}"] = s.detach().cpu().numpy()
    np.savez(path, **out)


def load(path, model, optimizer=None, build=None):
    data = np.load(path if str(path).endswith(".npz") else str(path) + ".npz", allow_pickle=False)
    if build is not None and _unbuilt(model):
        build()
    n_saved = sum(1 for k in data.files if k.startswith("var/"))
    variables = model.variables
    pending = _unbuilt(model)
    if pending or n_saved != len(variables):
        raise ValueError(f"checkpoint holds {n_saved} variables, the model has {len(variables)}"
                         + (f" ({pending} not built yet: call the model once, or pass build=)" if pending else ""))
    names = [str(x) for x in data["names"]] if "names" in data.files else None
    for k, v in enumerate(variables):
        a = data[f"var/{k}"]
        if names is not None and names[k] != v.name:
            raise ValueError(f"checkpoint variable {k} is {names[k]!r}, the model's is {v.name!r}")
        if tuple(a.shape) != tuple(v.shape):
            raise ValueError(f"checkpoint variable {k} has shape {a.shape}, model expects {tuple(v.shape)}")
        saved = str(data[f"dtype/{k}"]) if f"dtype/{k}" in data.files else "float32"
        if saved != _dtype(v):
            raise ValueError(f"checkpoint variable {k} ({v.name!r}) is {saved}, the model's is {_dtype(v)}")
    slots = []
    if optimizer is not None and "iterations" in data.files:
        # copy_ broadcasts: a row-wise [rows] accumulator would silently fill an element-wise [rows, dim] one
        for k, v in enumerate(variables):
            s = list(optimizer.slots(v))
            for j in range(2):
                key = f"slot{j}/{k}"
                if key in data.files and s[j] is not None:
                    if tuple(data[key].shape) != tuple(s[j].shape):
                        raise ValueError(f"checkpoint slot {key} of {v.name!r} has shape {data[key].shape}, "
                                         f"{type(optimizer).__name__} expects {tuple(s[j].shape)}")
                    slots.append((s[j], data[key]))
    for k, v in enumerate(variables):
        if _dtype(v) == "bfloat16":
            v.t.view(torch.int16).copy_(torch.from_numpy(data[f"var/{k}"].view(np.int16)))
        else:
            v.assign(data[f"var/{k}"])
    if optimizer is not None and "iterations" in data.files:
        optimizer.iterations = int(data["iterations"])
        for s, a in slots:
            s.copy_(torch.from_numpy(a))
