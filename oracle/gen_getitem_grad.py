"""Golden gradients of Tensor.__getitem__ from the REAL reference (the unmodified package oracle/stage_ref.py stages
into oracle/_ref/):

    python oracle/gen_getitem_grad.py   ->  tests/golden/getitem_grad.npz

For every case of oracle/getitem_cases.py whose key gives a value (errors are left to getitem.npz) and each dtype: the
gradients of sum(w * t[key].torch()) (of sum(w * t[key]) for a scalar) with respect to every core and every Tucker
factor, w drawn from a seed per case and stored beside them.  The Tucker tensors are rebuilt from the cores and factors
tests/golden/getitem.npz stores, so both sides index the same tensor."""
import os
import sys
import warnings
import zlib

import numpy as np

warnings.filterwarnings("ignore")
HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
sys.path.insert(0, REPO)

import torch  # noqa: E402

from oracle import getitem_cases as gc, stage_ref  # noqa: E402

stage_ref.stage()
tn = stage_ref.load()  # the real reference
if tn is None:
    raise SystemExit("gen_getitem_grad: the reference package is not staged under oracle/_ref")
gold = np.load(os.path.join(REPO, "tests", "golden", "getitem.npz"))


def leaves(spec, dname):
    """(cores, Us or None, batch) as fresh leaves that require grad."""
    t = gc.tensor(spec, gc.DTYPES[dname])
    if t is None:
        n = int(gold[f"{spec}/{dname}/n"])
        cores = [torch.tensor(gold[f"{spec}/{dname}/core{k}"]) for k in range(n)]
        Us = [torch.tensor(gold[f"{spec}/{dname}/U{k}"]).requires_grad_() for k in range(n)]
        return [c.requires_grad_() for c in cores], Us, False
    cores, _, batch = t
    return [c.clone().requires_grad_() for c in cores], None, batch


def weights(name, dname, shape, dtype):
    g = torch.Generator().manual_seed(zlib.crc32(f"{name}/{dname}".encode()))
    return torch.randn(tuple(shape), generator=g, dtype=torch.float64).to(dtype)


out = {}
for dname, dt in gc.DTYPES.items():
    for name, (spec, key) in gc.KEYS.items():
        if str(gold[f"{name}/{dname}/kind"]) not in ("tensor", "scalar"):
            continue
        cores, Us, batch = leaves(spec, dname)
        t = tn.Tensor(cores, Us=Us, batch=batch) if Us is not None else tn.Tensor(cores, batch=batch)
        r = t[key("cpu")]
        v = r.torch() if isinstance(r, tn.Tensor) else r
        w = weights(name, dname, v.shape, dt)
        (w * v).sum().backward()
        p = f"{name}/{dname}"
        out[f"{p}/w"] = w.numpy()
        for k, c in enumerate(cores):
            out[f"{p}/dcore{k}"] = (c.grad if c.grad is not None else torch.zeros_like(c)).numpy()
        for k, U in enumerate(Us or []):
            out[f"{p}/dU{k}"] = (U.grad if U.grad is not None else torch.zeros_like(U)).numpy()
        print(name, dname, [tuple(c.shape) for c in cores], flush=True)

np.savez_compressed(os.path.join(REPO, "tests", "golden", "getitem_grad.npz"), **out)
