"""Checkpoint / resume (absent from the reference, SURVEY §5).

Rank 0 writes ``{"model": state_dict, "optim": ..., "steps": ..}`` atomically
(tmp file + rename).  Works for ``nn.Module`` models and for the fused trainer
(which exposes ``state_dict()`` over its flat fp32 parameter/momentum buffers
using the reference's parameter names).  Momentum is always ALSO stored per
parameter name under ``"momentum"`` -- the one form both engines read -- so a
checkpoint written by the fused engine resumes on the torch engine (and vice
versa) with its momentum; a checkpoint whose momentum the loading side cannot
use raises a warning instead of silently training from zero momentum.

``FlatAdamW`` state is stored the same way, per parameter name under
``"optim_state"`` (``named_state()``: ``torch.optim.AdamW``'s per-parameter
form), so an AdamW checkpoint crosses world sizes and sharded / unsharded runs."""
from __future__ import annotations

import os
from typing import Any, Dict

import torch

__all__ = ["save_checkpoint", "load_checkpoint", "restore_optimizer"]


def save_checkpoint(path: str, model, optimizer=None, **extra: Any) -> str:
    """Atomically write ``model`` (module or fused trainer), ``optimizer`` state and ``extra`` keys to ``path``."""
    sd = model.state_dict()
    if "model" in sd and isinstance(sd.get("model"), dict):   # fused trainer: already structured
        blob: Dict[str, Any] = dict(sd)
    else:
        blob = {"model": {k: v.detach().cpu() for k, v in sd.items()}}
    if optimizer is not None:
        blob["optim"] = optimizer.state_dict()
        if "momentum" not in blob and hasattr(optimizer, "named_momentum"):
            blob["momentum"] = optimizer.named_momentum(model)        # canonical per-name form (see module docstring)
        if hasattr(optimizer, "named_state"):
            blob["optim_state"] = optimizer.named_state(model)        # FlatAdamW's per-name form
    blob.update(extra)
    tmp = f"{path}.tmp.{os.getpid()}"
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    torch.save(blob, tmp)
    os.replace(tmp, path)
    return path


def load_checkpoint(path: str, model=None, optimizer=None, map_location="cpu") -> Dict[str, Any]:
    """Restore ``model`` (an ``nn.Module`` or a fused trainer) and, when given, ``optimizer`` (``torch.optim`` or
    ``FlatSGD`` / ``FlatAdamW``) from ``path``; returns the whole blob (``steps``, ``history``, ...)."""
    blob = torch.load(path, map_location=map_location)
    if model is not None:
        if isinstance(model, torch.nn.Module):
            model.load_state_dict(blob["model"])
        else:                                   # fused trainer: parameters + momentum + step counter in one dict
            model.load_state_dict(blob)
    if optimizer is not None:
        restore_optimizer(optimizer, model, blob)
    return blob


def restore_optimizer(optimizer, model, blob: Dict[str, Any]) -> None:
    """Put the checkpoint's optimizer state into ``optimizer``: its own ``state_dict`` when the blob has one in a
    compatible layout, else the per-name momentum (a checkpoint from the other engine)."""
    import warnings
    optim = blob.get("optim")
    if optim is not None:
        try:
            optimizer.load_state_dict(optim)
            return
        except Exception as e:                     # different bucket layout / optimizer class: fall through to names
            warnings.warn(f"checkpoint optimizer state does not fit this optimizer ({e!r}); trying per-name momentum")
    named = blob.get("momentum")
    state = blob.get("optim_state")
    if state and hasattr(optimizer, "load_named_state") and model is not None:
        if optimizer.load_named_state(model, state) == 0:
            warnings.warn("checkpoint optimizer-state names match no parameter of this model: the state restarts at zero")
    elif named and hasattr(optimizer, "load_named_momentum") and model is not None:
        if optimizer.load_named_momentum(model, named) == 0:
            warnings.warn("checkpoint momentum names match no parameter of this model: momentum restarts at zero")
    elif named or state or optim is not None:
        warnings.warn("checkpoint carries momentum this optimizer cannot read: momentum restarts at zero")
