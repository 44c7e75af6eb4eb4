"""Loader for the committed golden vectors (tests/golden/*.npz, produced by
tests/golden/gen_golden.py from the unmodified reference)."""
import glob
import json
import os

import numpy as np
import torch

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


class Case:
    def __init__(self, path):
        self.name = os.path.splitext(os.path.basename(path))[0]
        z = np.load(path)
        self.meta = json.loads(str(z["meta"]))
        self.ins, self.sd, self.outs = {}, {}, {}
        for key in z.files:
            if key == "meta":
                continue
            grp, name = key.split(".", 1)
            t = torch.from_numpy(z[key])
            {"in": self.ins, "sd": self.sd, "out": self.outs}[grp][name] = t
        for name, (seed, shape) in self.meta.get("seeded", {}).items():
            self.sd[name] = seeded_weight(seed, shape)

    def __repr__(self):
        return self.name


def seeded_weight(seed, shape):
    """A large weight of a golden model, not stored but drawn from its seed (keeps every golden file small):
    normal with std 1/sqrt(fan_in)."""
    g = torch.Generator().manual_seed(seed)
    fan_in = max(1, int(np.prod(shape[1:])))
    return torch.randn(*shape, generator=g) / float(np.sqrt(fan_in))


def names(prefix):
    return sorted(os.path.splitext(os.path.basename(p))[0]
                  for p in glob.glob(os.path.join(GOLDEN_DIR, prefix + "*.npz")))


def load(name):
    return Case(os.path.join(GOLDEN_DIR, name + ".npz"))


def dense_params(case, prefix="gconv.nn."):
    """Functional parameter dict (oracle.dense.basic_conv) from a golden state_dict."""
    sd, meta = case.sd, case.meta
    p = {"weight": sd[prefix + "0.weight"]}
    if prefix + "0.bias" in sd:
        p["bias"] = sd[prefix + "0.bias"]
    nxt = 1
    if meta.get("act") not in (None, "none"):
        if meta["act"] == "prelu":
            p["slope"] = sd[prefix + "1.weight"]
        nxt = 2
    if meta.get("norm") == "batch":
        p["norm"] = {k: sd["%s%d.%s" % (prefix, nxt, k)]
                     for k in ("weight", "bias", "running_mean", "running_var")}
    return p
