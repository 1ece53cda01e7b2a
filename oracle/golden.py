"""ORACLE (test infrastructure) — reading and writing tests/golden/.

A golden is one torch.save file, or, when it would exceed 1 MB, a directory of the same name whose
parts (`00.pt`, `01.pt`, ...) are concatenated (lists) or merged (dicts) in file-name order."""
from __future__ import annotations

import os
import shutil

import torch


def load(golden_dir: str, name: str):
    path = os.path.join(golden_dir, name)
    if os.path.isfile(path):
        return torch.load(path, weights_only=False)
    obj = None
    for part in sorted(os.listdir(path)):
        p = torch.load(os.path.join(path, part), weights_only=False)
        if obj is None:
            obj = p
        elif isinstance(obj, list):
            obj.extend(p)
        else:
            obj.update(p)
    return obj


def save_parts(golden_dir: str, name: str, parts) -> None:
    path = os.path.join(golden_dir, name)
    if os.path.isfile(path):
        os.remove(path)
    shutil.rmtree(path, ignore_errors=True)
    os.makedirs(path)
    for i, p in enumerate(parts):
        torch.save(p, os.path.join(path, f"{i:02d}.pt"))
