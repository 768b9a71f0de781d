"""Golden vectors for Tensor.__getitem__ (tensor.py:1019-1434) from the REAL reference, the unmodified package that
oracle/stage_ref.py stages into oracle/_ref/.

    python oracle/gen_getitem.py   ->  tests/golden/getitem.npz

Per case and dtype (oracle/getitem_cases.py): the result's kind ("scalar", "tensor", or the exception the key raises), its values (the dense result of
a Tensor, the value of a scalar), and for a Tensor its core and Tucker factor shapes.  The cores and factors of the
Tucker tensors the reference's constructor built are stored once per spec and dtype; the other tensors are rebuilt from
their seeds."""
import os
import sys
import warnings

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
    raise SystemExit("gen_getitem: the reference package is not staged under oracle/_ref")

out = {}
built = {}
for dname, dt in gc.DTYPES.items():
    for spec, (kind, _) in gc.SPECS.items():
        if kind == "tucker":
            dense, rt, rtt = gc.dense_for(spec, dt)
            t = tn.Tensor(dense, ranks_tucker=list(rt), ranks_tt=rtt)
            for k, c in enumerate(t.cores):
                out[f"{spec}/{dname}/core{k}"] = c.detach().numpy()
                out[f"{spec}/{dname}/U{k}"] = t.Us[k].detach().numpy()
            out[f"{spec}/{dname}/n"] = np.int64(len(t.cores))
        else:
            cores, Us, batch = gc.tensor(spec, dt)
            t = tn.Tensor(cores, batch=batch)
        built[spec, dname] = t
    for name, (spec, key) in gc.KEYS.items():
        t = built[spec, dname]
        p = f"{name}/{dname}"
        try:
            r = t[key("cpu")]
        except (IndexError, ValueError) as e:
            out[f"{p}/kind"] = np.array(type(e).__name__)
            print(name, dname, type(e).__name__, flush=True)
            continue
        if isinstance(r, tn.Tensor):
            out[f"{p}/kind"] = np.array("tensor")
            out[f"{p}/value"] = r.torch().detach().numpy()
            out[f"{p}/core_shapes"] = np.array([list(c.shape) + [0] * (4 - c.dim()) for c in r.cores], dtype=np.int64)
            out[f"{p}/U_shapes"] = np.array([list(U.shape) + [0] * (3 - U.dim()) if U is not None else [-1, -1, -1]
                                             for U in r.Us], dtype=np.int64)
        else:
            out[f"{p}/kind"] = np.array("scalar")
            out[f"{p}/value"] = r.detach().numpy()
        print(name, dname, out[f"{p}/kind"], np.asarray(out[f"{p}/value"]).shape, flush=True)

np.savez_compressed(os.path.join(REPO, "tests", "golden", "getitem.npz"), **out)
