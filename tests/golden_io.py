"""Loader of the render goldens tests/golden/*.pt.  A golden whose per-node per-sample tensors would make one file large keeps
them beside it, one file per node (tests/golden/<name>/<node>.pt); load() puts them back under rec["nodes"]."""
import os

import torch


def load(path):
    rec = torch.load(path)
    if "nodes" not in rec:
        d = path[:-3]
        rec["nodes"] = {nid: torch.load(os.path.join(d, f"{nid}.pt")) for nid in rec["scene_kwargs"]["nodes"]}
    return rec
