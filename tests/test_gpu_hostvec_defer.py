"""Host-vector SpMV with deferred completion (B200SP_SPMV_OPT_HOSTVEC_DEFER, spmv.cu): a call no longer makes the stream wait for
its own download of y, so upload, kernel and download of consecutive calls overlap; b200sp_spmv_hostvec_flush + a stream
synchronisation complete all of them.  Results must be the bits of the stream-ordered mode, call by call, with distinct and with
shared host buffers."""
import numpy as np
import pytest
import torch

from helpers import kk_matrix

pytestmark = pytest.mark.gpu


def test_hostvec_deferred_completion(cuda):
    from kokkos_kernels_b200 import sparse as sp

    n = 300000
    rp, ci, v = kk_matrix(n, n, n * 40, 5, 3000)  # nnz >= 2^22: the pipelined path
    assert len(ci) >= (1 << 22)
    t = lambda a: torch.from_numpy(a).to(cuda)
    A = sp.CrsMatrix(t(rp), t(ci), t(v), n)
    rng = np.random.default_rng(1)
    calls = 7
    xs = [torch.from_numpy(rng.uniform(-1, 1, n)).pin_memory() for _ in range(calls)]
    ref = []
    h = sp.SPMVHandle()
    for x in xs:  # stream-ordered mode: the reference bits
        y = torch.empty(n, dtype=torch.float64).pin_memory()
        sp.spmv_hostvec(h, "N", 1.5, A, x, 0.0, y)
        torch.cuda.synchronize()
        ref.append(y.clone())
    h.hostvec_defer(True)
    ys = [torch.full((n,), float("nan"), dtype=torch.float64).pin_memory() for _ in range(calls)]
    for x, y in zip(xs, ys):
        sp.spmv_hostvec(h, "N", 1.5, A, x, 0.0, y)
    with pytest.raises((sp.B200SparseError, sp.B200SparseInvalidArgument)):
        h.hostvec_defer(False)  # downloads outstanding
    h.hostvec_flush()
    torch.cuda.synchronize()
    for y, r in zip(ys, ref):
        assert torch.equal(y, r)
    # one shared y buffer (what bench.py does): the last call's result stands
    yshared = torch.empty(n, dtype=torch.float64).pin_memory()
    for x in xs:
        sp.spmv_hostvec(h, "N", 1.5, A, x, 0.0, yshared)
    h.hostvec_flush()
    torch.cuda.synchronize()
    assert torch.equal(yshared, ref[-1])
    # beta != 0 with distinct buffers: y is uploaded at call time
    y0 = [torch.from_numpy(rng.uniform(-1, 1, n)).pin_memory() for _ in range(3)]
    exp = []
    h.hostvec_defer(False)
    for x, y in zip(xs, y0):
        yy = y.clone().pin_memory()
        sp.spmv_hostvec(h, "N", 2.0, A, x, -0.5, yy)
        torch.cuda.synchronize()
        exp.append(yy.clone())
    h.hostvec_defer(True)
    yd = [y.clone().pin_memory() for y in y0]
    for x, y in zip(xs, yd):
        sp.spmv_hostvec(h, "N", 2.0, A, x, -0.5, y)
    h.hostvec_flush()
    torch.cuda.synchronize()
    for y, r in zip(yd, exp):
        assert torch.equal(y, r)
    h.hostvec_defer(False)
