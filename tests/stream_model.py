"""Python restatement of the streamed step 0's chunk plan (csrc/sweep.cuh make_chunk_plan) and of tn.Tensor's
stream-or-copy rule (ops.stream_instead_of_copy), for the CPU tests and the GPU tests' expected chunk counts."""

PROJ_TC_MIN_ROWS = 16384
DEFAULT_CHUNK = 256 << 20


def chunk_plan(rows, n, row_bytes, chunk_bytes, proj_tc, kb_inner):
    """(unit, min_rows, chunk_rows, nchunks, last_rows) for a (rows x n) step 0: chunks of whole `unit`-row blocks (lcm of
    16, the narrow Gram's fold and 8 inner for a K-blocked carry), at least PROJ_TC_MIN_ROWS rows when the projection is
    on the tensor cores and never fewer than n; a last piece shorter than that joins the chunk before it."""
    unit = 8 * kb_inner if kb_inner else 16
    min_rows = max(PROJ_TC_MIN_ROWS if proj_tc else 1, n)
    chunk_bytes = chunk_bytes or DEFAULT_CHUNK
    chunk_rows = max(chunk_bytes // row_bytes // unit * unit, -(-min_rows // unit) * unit)
    if chunk_rows >= rows:
        return unit, min_rows, rows, 1, rows
    nch = -(-rows // chunk_rows)
    last = rows - (nch - 1) * chunk_rows
    if last < min_rows:
        nch, last = nch - 1, last + chunk_rows
    return unit, min_rows, chunk_rows, nch, last


def streams(input_bytes, workspace_bytes, free_bytes):
    """tn.Tensor(X_cpu, ranks_tt=r) streams when the device image plus the device call's workspace exceeds free memory."""
    return input_bytes + workspace_bytes > free_bytes
