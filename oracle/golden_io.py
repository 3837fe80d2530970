"""Store / load nested results of the reference (tensors, arrays, lists, tuples, dicts, None, scalars) as one .npz file.

The structure goes into the `__meta__` entry as JSON; every tensor or array becomes one npz entry, with its dtype kept (a tensor
comes back as a tensor, an array as an array).  Used by oracle/make_golden_live.py to write tests/golden/live/*.npz and by the
tests that read them."""
import json

import numpy as np


def _pack(obj, store):
    import torch
    if obj is None:
        return None
    if torch.is_tensor(obj):
        key = f"a{len(store)}"
        store[key] = obj.detach().cpu().numpy()
        return {"t": key}
    if isinstance(obj, np.ndarray):
        key = f"a{len(store)}"
        store[key] = obj
        return {"n": key}
    if isinstance(obj, (list, tuple)):
        return {"l" if isinstance(obj, list) else "u": [_pack(x, store) for x in obj]}
    if isinstance(obj, dict):
        return {"d": [[k, _pack(v, store)] for k, v in obj.items()]}
    if isinstance(obj, (bool, int, float, str)):
        return {"v": obj, "type": type(obj).__name__}
    if isinstance(obj, np.generic):
        return {"v": obj.item(), "type": "np." + type(obj).__name__}
    raise TypeError(f"cannot store {type(obj)}")


def _unpack(desc, data):
    import torch
    if desc is None:
        return None
    if "t" in desc:
        return torch.from_numpy(np.array(data[desc["t"]]))
    if "n" in desc:
        return np.array(data[desc["n"]])
    if "l" in desc:
        return [_unpack(x, data) for x in desc["l"]]
    if "u" in desc:
        return tuple(_unpack(x, data) for x in desc["u"])
    if "d" in desc:
        return {k: _unpack(v, data) for k, v in desc["d"]}
    t = desc["type"]
    if t.startswith("np."):
        return getattr(np, t[3:])(desc["v"])
    return {"bool": bool, "int": int, "float": float, "str": str}[t](desc["v"])


def save(path, obj):
    store = {}
    meta = _pack(obj, store)
    np.savez_compressed(path, __meta__=np.array(json.dumps(meta)), **store)


def load(path):
    with np.load(path, allow_pickle=False) as data:
        return _unpack(json.loads(str(data["__meta__"])), data)
