"""The tensors and keys of tests/golden/getitem.npz (oracle/gen_getitem.py), shared with the tests that replay them.

tensor(spec, dtype) -> (cores, Us, batch) as CPU torch tensors built from seeds; KEYS maps a case name to
(tensor spec, dtype, key builder); a key builder takes the torch module of the cores' device ("cpu" for the reference)
so that torch-tensor keys can be made on either side."""
import numpy as np
import torch

f64, f32 = torch.float64, torch.float32


def _tt(seed, shape, ranks, dtype, batch=None):
    g = torch.Generator().manual_seed(seed)
    r = [1] + list(ranks) + [1]
    lead = [] if batch is None else [batch]
    return [torch.randn(*lead, r[k], shape[k], r[k + 1], generator=g, dtype=dtype) for k in range(len(shape))]


def _dense(seed, shape, dtype):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g, dtype=dtype)


S4 = (4, 5, 6, 3)
# spec -> (kind, args); "tucker" / "tt_tucker" are built by the reference's constructor from a dense tensor, so they are
# stored as the cores and factors the reference made (gen_getitem.py), not rebuilt here
SPECS = {
    "tt": ("tt", (1, S4, (3, 4, 2))),
    "one_mode": ("tt", (2, (9,), ())),
    "unit_modes": ("tt", (3, (1, 3, 1, 4), (2, 2, 3))),
    "rank1": ("tt", (4, (3, 4, 5), (1, 1))),
    "tucker": ("tucker", (5, S4, None)),
    "tt_tucker": ("tucker", (6, S4, 2)),
    "cp": ("cp", (7, S4, 3)),
    "batch": ("batch", (8, S4, (3, 2, 2), 3)),
}


def tensor(spec, dtype):
    """(cores, Us, batch) of a spec whose cores come from seeds; None for the Tucker specs."""
    kind, a = SPECS[spec]
    if kind == "tt":
        return _tt(a[0], a[1], a[2], dtype), None, False
    if kind == "cp":
        g = torch.Generator().manual_seed(a[0])
        return [torch.randn(n, a[2], generator=g, dtype=dtype) for n in a[1]], None, False
    if kind == "batch":
        return _tt(a[0], a[1], a[2], dtype, batch=a[3]), None, True
    return None


def dense_for(spec, dtype):
    """The dense input of a Tucker spec: tn.Tensor(dense, ranks_tucker=(2, 3, 3, 2)[, ranks_tt=2])."""
    kind, a = SPECS[spec]
    return _dense(a[0], a[1], dtype), (2, 3, 3, 2), a[2]


_Xs = np.array([[0, 1, 2, 0], [3, 4, 5, 2], [1, 0, 0, 1], [2, 2, 3, 0], [3, 1, 4, 2], [0, 4, 1, 1], [1, 3, 5, 2]])

# name -> (spec, key(device))
KEYS = {
    "int": ("tt", lambda d: (1, 2, 3, 0)),
    "int_negative": ("tt", lambda d: (-1, 2, -3, 1)),
    "matrix_numpy": ("tt", lambda d: _Xs.copy()),
    "matrix_torch": ("tt", lambda d: torch.tensor(_Xs, device=d)),
    "lists": ("tt", lambda d: ([0, 1, 3], [2, 2, 4], [5, 0, 1], [1, 2, 0])),
    "list_mode0": ("tt", lambda d: [3, 0, 2, 2]),
    "slices_steps": ("tt", lambda d: (slice(0, 4, 2), slice(1, None), slice(None, None, 3), slice(None))),
    "none_ellipsis": ("tt", lambda d: (None, 1, Ellipsis, None)),
    "ellipsis_int": ("tt", lambda d: (Ellipsis, 2)),
    "inner_block": ("tt", lambda d: (slice(None), [0, 2, 4, 1], [1, 3, 5, 0], slice(1, 3))),
    "inner_block_torch": ("tt", lambda d: (slice(None), torch.tensor([0, 2, 4, 1], device=d),
                                           torch.tensor([1, 3, 5, 0], device=d), slice(None))),
    "int_slice_int_slice": ("tt", lambda d: (1, slice(None), 2, slice(0, 2))),
    "slice_int_slice_int": ("tt", lambda d: (slice(None), 2, slice(None), 1)),
    "ints_then_slice": ("tt", lambda d: (1, 2, slice(None), 0)),
    "int_then_block": ("tt", lambda d: (1, [0, 2], [3, 4], slice(None))),
    "block_then_int": ("tt", lambda d: ([0, 1], [2, 3], 1, slice(None))),
    "block_then_ints": ("tt", lambda d: (slice(1, 3), [0, 4], 1, 2)),
    "one_mode_int": ("one_mode", lambda d: (3,)),
    "one_mode_list": ("one_mode", lambda d: ([1, 4, 8],)),
    "one_mode_slice": ("one_mode", lambda d: (slice(2, 7, 2),)),
    "unit_block": ("unit_modes", lambda d: (0, [1, 2], [0, 0], [3, 0])),
    "not_contiguous": ("unit_modes", lambda d: (0, [1, 2], 0, [3, 0])),
    "unequal_lengths": ("tt", lambda d: ([0, 1], [2, 3, 4], 0, 0)),
    "too_many": ("tt", lambda d: (0, 0, 0, 0, 0)),
    "unit_mixed": ("unit_modes", lambda d: (0, slice(None), 0, 2)),
    "rank1_int": ("rank1", lambda d: (1, 2, 3)),
    "rank1_matrix": ("rank1", lambda d: np.array([[0, 1, 2], [2, 3, 4], [1, 0, 0]])),
    "tucker_int": ("tucker", lambda d: (1, 2, 3, 0)),
    "tucker_matrix": ("tucker", lambda d: _Xs.copy()),
    "tucker_block": ("tucker", lambda d: (slice(None), [0, 2, 4], [1, 3, 5], slice(None))),
    "tucker_int_slice": ("tucker", lambda d: (1, slice(1, 4), 2, slice(None))),
    "tt_tucker_int": ("tt_tucker", lambda d: (3, 0, 5, 2)),
    "tt_tucker_matrix": ("tt_tucker", lambda d: _Xs.copy()),
    "tt_tucker_mixed": ("tt_tucker", lambda d: (slice(None, None, 2), [1, 4], [0, 5], 1)),
    "cp_int": ("cp", lambda d: (1, 2, 3, 0)),
    "cp_matrix": ("cp", lambda d: _Xs.copy()),
    "cp_mixed": ("cp", lambda d: (slice(None), [0, 2, 4], [1, 3, 5], 2)),
    "batch_slice_block": ("batch", lambda d: (slice(0, 2), slice(None), [0, 2, 4], [1, 3, 5], slice(None))),
    "batch_slice_ints": ("batch", lambda d: (slice(None), 1, slice(None), 2, 0)),
    "batch_int": ("batch", lambda d: (1, [0, 3], [1, 4], 2, slice(None))),
    "batch_int_all_int": ("batch", lambda d: (2, 1, 2, 3, 0)),
}
DTYPES = {"f64": f64, "f32": f32}
