"""The seeded cases of tests/golden/attention_*.npz (make_golden_attention.py) that the CPU and GPU tests of the standalone
Attention module share; the module itself is restated by oracle.flowtron_oracle.attention_forward.

Inputs and weights are regenerated from each case's seed with torch's CPU generator; the fixtures carry their sums so a test
knows it runs on exactly what the reference ran on."""
from __future__ import annotations

import math
import os
from typing import Optional

import torch
from torch import Tensor

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
PRE = ("query", "key", "value", "v")

# Dq, E, A: the default constructor and the AR_Step dimensions
DIMS = {"default": (80, 640, 128), "ar_step": (1024, 640, 640)}

# name -> dims, B, T, L, valid keys per row (None: no mask), prior, temperature, attn given, keys != values, seed
CASES = {
    "default_nomask":      dict(dims="default", B=3, T=65, L=160, lens=None, prior=False, temp=1.0, given=False, kv=False, seed=11),
    "default_ragged":      dict(dims="default", B=3, T=65, L=160, lens=[160, 97, 1], prior=False, temp=1.0, given=False, kv=False, seed=12),
    "default_prior":       dict(dims="default", B=3, T=65, L=160, lens=[160, 97, 1], prior=True, temp=1.0, given=False, kv=False, seed=13),
    "default_temp":        dict(dims="default", B=1, T=65, L=160, lens=[131], prior=False, temp=1.7, given=False, kv=False, seed=14),
    "default_given":       dict(dims="default", B=3, T=65, L=160, lens=None, prior=False, temp=1.0, given=True, kv=False, seed=15),
    "default_kv":          dict(dims="default", B=3, T=65, L=160, lens=[160, 50, 7], prior=False, temp=1.0, given=False, kv=True, seed=16),
    "default_b40":         dict(dims="default", B=40, T=1, L=160, lens="random", prior=False, temp=1.0, given=False, kv=False, seed=17),
    "default_t1000":       dict(dims="default", B=1, T=1000, L=1, lens=None, prior=False, temp=1.0, given=False, kv=False, seed=18),
    "default_l1024_prior": dict(dims="default", B=1, T=1, L=1024, lens=[1000], prior=True, temp=1.0, given=False, kv=False, seed=19),
    "ar_ragged":           dict(dims="ar_step", B=1, T=65, L=160, lens=[113], prior=False, temp=1.0, given=False, kv=False, seed=21),
    "ar_prior_temp":       dict(dims="ar_step", B=1, T=65, L=160, lens=[160], prior=True, temp=1.7, given=False, kv=False, seed=22),
    "ar_given":            dict(dims="ar_step", B=1, T=65, L=160, lens=None, prior=False, temp=1.0, given=True, kv=True, seed=23),
    "ar_l700":             dict(dims="ar_step", B=1, T=1, L=700, lens=[523], prior=False, temp=1.0, given=False, kv=False, seed=24),
    "ar_l1024":            dict(dims="ar_step", B=1, T=1, L=1024, lens=None, prior=False, temp=1.0, given=False, kv=True, seed=25),
}


def case_lens(c: dict) -> Optional[Tensor]:
    if c["lens"] is None:
        return None
    if c["lens"] == "random":
        g = torch.Generator().manual_seed(c["seed"] + 1)
        return torch.randint(1, c["L"] + 1, (c["B"],), generator=g)
    return torch.tensor(c["lens"])


def case_inputs(c: dict) -> dict:
    """Weights (state_dict of the module) and inputs of a case, fp32 on the CPU.  Weights are Xavier-scaled (gain 5/3, the
    module's w_init_gain='tanh') normals."""
    Dq, E, A = DIMS[c["dims"]]
    B, T, L = c["B"], c["T"], c["L"]
    g = torch.Generator().manual_seed(c["seed"])
    W = {}
    for name, (o, i) in zip(PRE, ((A, Dq), (A, E), (A, E), (1, A))):
        W[f"{name}.linear_layer.weight"] = torch.randn(o, i, generator=g) * (5.0 / 3.0) * math.sqrt(2.0 / (i + o))
    x = dict(W=W, queries=torch.randn(T, B, Dq, generator=g), keys=torch.randn(L, B, E, generator=g))
    x["values"] = torch.randn(L, B, E, generator=g) if c["kv"] else x["keys"]
    lens = case_lens(c)
    x["lens"] = lens
    x["mask"] = None if lens is None else ~(torch.arange(L)[None, :] < lens[:, None])[..., None]
    x["prior"] = torch.softmax(2.0 * torch.randn(B, T, L, generator=g), dim=2) if c["prior"] else None
    x["attn"] = torch.softmax(3.0 * torch.randn(B, T, L, generator=g), dim=2) if c["given"] else None
    return x


def input_sums(x: dict) -> dict:
    """float64 sums of every generated tensor (fixture check that the inputs regenerate exactly)."""
    out = {f"sum/{k}": float(v.double().sum()) for k, v in x["W"].items()}
    for k in ("queries", "keys", "values", "prior", "attn"):
        if x[k] is not None:
            out[f"sum/{k}"] = float(x[k].double().sum())
    return out
