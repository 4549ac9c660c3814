"""Checkpoint / resume for the parameter server.

The reference keeps the global model and ``loss_history`` only in manager RAM
(manager.py:24, update_manager.py:21): a manager restart loses the job.  Here
``Experiment.end_round`` can persist

    {"state_dict", "n_updates", "loss_history", "update_name", "name", "format"}

with ``torch.save``, plus ``"server_opt": {"config", "m", "v"}`` when the experiment runs a server optimizer.
``state_dict`` is the plain PyTorch layout (name -> tensor
in module order), so ``torch.load(path)["state_dict"]`` drops straight into a
stock ``nn.Module.load_state_dict`` -- the same layout the reference ships on
the wire (manager.py:78).  Writes are atomic (tmp + rename) and the last
``keep`` files are retained.
"""
from __future__ import annotations

import glob
import os
import re
import tempfile
from collections import OrderedDict
from typing import Optional

import torch

FORMAT = "baton_b200.ckpt.v1"


def _cpu_state_dict(model_or_sd) -> "OrderedDict[str, torch.Tensor]":
    sd = model_or_sd.state_dict() if hasattr(model_or_sd, "state_dict") else model_or_sd
    return OrderedDict((k, v.detach().to("cpu").clone()) for k, v in sd.items())


def save_checkpoint(directory: str, name: str, model, update_manager, *, keep: int = 3,
                    server_opt: Optional[dict] = None) -> str:
    os.makedirs(directory, exist_ok=True)
    snap = update_manager.snapshot()
    payload = {
        "format": FORMAT,
        "name": name,
        "state_dict": _cpu_state_dict(model),
        "n_updates": snap["n_updates"],
        "loss_history": snap["loss_history"],
        "update_name": snap["update_name"],
    }
    if server_opt is not None:
        payload["server_opt"] = server_opt
    final = os.path.join(directory, "{}_{:05d}.pt".format(name, snap["n_updates"]))
    fd, tmp = tempfile.mkstemp(dir=directory, suffix=".tmp")
    os.close(fd)
    try:
        torch.save(payload, tmp)
        os.replace(tmp, final)
    finally:
        if os.path.exists(tmp):
            os.unlink(tmp)
    if keep and keep > 0:
        for old in list_checkpoints(directory, name)[:-keep]:
            try:
                os.unlink(old)
            except OSError:
                pass
    return final


def list_checkpoints(directory: str, name: str):
    pat = re.compile(r"^{}_(\d+)\.pt$".format(re.escape(name)))
    found = []
    for path in glob.glob(os.path.join(directory, "{}_*.pt".format(name))):
        m = pat.match(os.path.basename(path))
        if m:
            found.append((int(m.group(1)), path))
    return [p for _, p in sorted(found)]


def latest_checkpoint(directory: str, name: str) -> Optional[str]:
    ckpts = list_checkpoints(directory, name)
    return ckpts[-1] if ckpts else None


def load_checkpoint(path: str, model=None, update_manager=None, *, strict: bool = True) -> dict:
    payload = torch.load(path, map_location="cpu", weights_only=True)
    if payload.get("format") != FORMAT:
        raise ValueError("{} is not a {} file".format(path, FORMAT))
    if model is not None:
        model.load_state_dict(payload["state_dict"], strict=strict)
    if update_manager is not None:
        update_manager.restore(payload)
    return payload
