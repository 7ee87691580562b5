"""Reading a local safetensors checkpoint directory into a mirror's parameters (the `from_pretrained` of the DiT and the encoders)."""
from __future__ import annotations

import json
import os
from typing import Callable

import torch.nn as nn

from ._lib import CEError


def load_safetensors(model: nn.Module, root: str, weights_name: str, skip: Callable[[str], bool] = lambda k: False) -> None:
    """Copy `<root>/<weights_name>.safetensors`, or every shard `<weights_name>.safetensors.index.json` lists, into the parameters of
    `model`, each cast to its parameter's dtype.  A key the model does not have and a parameter no file holds are errors; keys for
    which `skip(key)` holds are ignored.  Local paths only (no hub download)."""
    from safetensors import safe_open

    index = os.path.join(root, weights_name + ".safetensors.index.json")
    if os.path.exists(index):
        with open(index) as f:
            files = sorted(set(json.load(f)["weight_map"].values()))
    else:
        files = [weights_name + ".safetensors"]
    params = dict(model.named_parameters())
    seen = set()
    for fn in files:
        with safe_open(os.path.join(root, fn), framework="pt", device="cpu") as sf:
            for k in sf.keys():
                if skip(k):
                    continue
                if k not in params:
                    raise CEError(f"unexpected key in checkpoint: {k}")
                params[k].data.copy_(sf.get_tensor(k).reshape(params[k].shape))
                seen.add(k)
    missing = sorted(set(params) - seen)
    if missing:
        raise CEError(f"checkpoint is missing {len(missing)} parameters, first: {missing[0]}")
