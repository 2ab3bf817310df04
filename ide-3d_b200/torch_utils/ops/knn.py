"""k-nearest-neighbour distances of the precision / recall metric (metrics/precision_recall.py) on sm_90a.

    kth_dist(rows [R, D], cols [C, D], kth) -> [R] fp32   the kth smallest |rows[r] - cols[c]| over c (the row's own zero distance
                                                          counts when rows is a slice of cols: the reference's kthvalue(nhood_size + 1))
    within(probes [Q, D], manifold [M, D], radius [M]) -> [Q] bool   any j with |probes[q] - manifold[j]| <= radius[j]

Features are CUDA fp16 with D a multiple of 8; each call is one tensor-core pass (ide3d_knn_kth_dist / ide3d_knn_within) that never
stores the distance matrix.  Distances are compared squared: |x|^2 + |y|^2 - 2 x.y with fp32 accumulation, clamped at 0.
"""

import torch

from ... import _lib as L


def _features(name, x):
    L.require_cuda(x)
    if x.dtype != torch.float16 or x.ndim != 2:
        raise RuntimeError(f'ide3d_b200.knn: {name} must be a 2-D float16 tensor, got {tuple(x.shape)} {x.dtype}')
    return x.contiguous()


def _scratch(nbytes, device):
    """The caller-owned scratch (the caching allocator's blocks are 512-byte aligned); None for sizes the entry point will refuse."""
    return None if nbytes < 0 else torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device=device)


def _nbytes(t):
    return 0 if t is None else t.numel()


def kth_dist(rows, cols, kth):
    rows, cols = _features('rows', rows), _features('cols', cols)
    if rows.device != cols.device or rows.shape[1] != cols.shape[1]:
        raise RuntimeError(f'ide3d_b200.knn: rows {tuple(rows.shape)} on {rows.device} and cols {tuple(cols.shape)} on {cols.device} differ')
    R, C, D = rows.shape[0], cols.shape[0], rows.shape[1]
    out = torch.empty(R, dtype=torch.float32, device=rows.device)
    lib = L.get_lib()
    with torch.cuda.device(rows.device):
        nbytes = lib.ide3d_knn_kth_dist_scratch_bytes(R, C, int(kth))
    scratch = _scratch(nbytes, rows.device)
    L.check(lib.ide3d_knn_kth_dist(rows.data_ptr(), R, cols.data_ptr(), C, D, int(kth), out.data_ptr(), L.ptr(scratch), _nbytes(scratch),
                                   L.stream_ptr(rows.device)))
    return out


def within(probes, manifold, radius):
    probes, manifold = _features('probes', probes), _features('manifold', manifold)
    L.require_cuda(radius)
    if probes.device != manifold.device or probes.shape[1] != manifold.shape[1] or radius.shape != (manifold.shape[0],):
        raise RuntimeError(f'ide3d_b200.knn: probes {tuple(probes.shape)}, manifold {tuple(manifold.shape)} and radius '
                           f'{tuple(radius.shape)} do not match')
    radius = radius.to(device=probes.device, dtype=torch.float32).contiguous()
    Q, M, D = probes.shape[0], manifold.shape[0], probes.shape[1]
    flags = torch.empty(Q, dtype=torch.uint8, device=probes.device)
    lib = L.get_lib()
    scratch = _scratch(lib.ide3d_knn_within_scratch_bytes(Q, M), probes.device)
    L.check(lib.ide3d_knn_within(probes.data_ptr(), Q, manifold.data_ptr(), M, D, radius.data_ptr(), flags.data_ptr(), L.ptr(scratch),
                                 _nbytes(scratch), L.stream_ptr(probes.device)))
    return flags.bool()
