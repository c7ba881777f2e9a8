"""Thin typed wrapper over the C-ABI: torch tensors are only device-memory holders
(``tensor.data_ptr()``), no torch op computes anything on the hot path."""
from __future__ import annotations

import contextlib
import ctypes as C

import numpy as np
import torch

from . import _abi


def _p(t, dtype=None):
    """device pointer of a tensor (None -> NULL); the dtype is asserted because the C-ABI
    takes raw pointers and would silently misread anything else."""
    if t is None:
        return C.c_void_p(0)
    if dtype is not None and t.dtype != dtype:
        raise TypeError("expected a %s tensor, got %s" % (dtype, t.dtype))
    if not t.is_cuda:
        raise TypeError("expected a CUDA tensor")
    if t.dim() > 1 and t.stride(-1) != 1:
        raise TypeError("innermost dimension must be contiguous")
    return C.c_void_p(t.data_ptr())


_F32, _I32, _I64, _F64 = torch.float32, torch.int32, torch.int64, torch.float64


def round_up(x, m):
    return (x + m - 1) // m * m


class DeviceCSR:
    """CSR matrix resident in HBM: indptr int64, indices int32, values float32 (float64 for the item-to-item matrix of
    ``Engine.cooc_build_csr``, which only ``Engine.i2i_topk_csr`` reads).  ``n_panels > 1``: panel-major storage
    (``pb200_csr_block_columns``): indptr has n_panels * n_rows + 1 entries, ``panel_ptr`` is the host array of panel
    offsets."""

    __slots__ = ("indptr", "indices", "values", "shape", "n_panels", "panel_cols", "panel_ptr")

    def __init__(self, indptr, indices, values, shape, n_panels=1, panel_cols=None, panel_ptr=None):
        self.indptr, self.indices, self.values, self.shape = indptr, indices, values, tuple(int(s) for s in shape)
        self.n_panels = int(n_panels)
        self.panel_cols = int(self.shape[1] if panel_cols is None else panel_cols)
        self.panel_ptr = panel_ptr          # ctypes int64 array (host) or None

    @property
    def nnz(self):
        return int(self.indices.shape[0])

    def view(self):
        """the ``pb200_csr_view`` struct for the C-ABI (holds raw pointers: keep ``self`` alive while it is used).  Its
        values are float32: every entry point that takes a view reads them so."""
        if self.values.dtype != torch.float32:
            raise TypeError("a pb200_csr_view holds float32 values, got %s" % self.values.dtype)
        return _abi.CsrView(self.shape[0], self.shape[1], self.nnz, self.indptr.data_ptr(), self.indices.data_ptr(),
                            self.values.data_ptr(), self.n_panels, self.panel_cols,
                            C.cast(self.panel_ptr, C.c_void_p) if self.panel_ptr is not None else None)

    def nbytes(self):
        return self.indptr.numel() * 8 + self.indices.numel() * 4 + self.values.numel() * self.values.element_size()


class _StreamFollowingLib:
    """Every C-ABI call runs on torch's CURRENT stream of the engine's device: tensors are allocated, uploaded and waited
    for relative to that stream (``torch.cuda.current_stream``), so the library context must enqueue on the same one.  When
    the current stream changed since the last call (``with torch.cuda.stream(s):``), the context is re-pointed first."""

    def __init__(self, lib, engine):
        self._lib, self._engine = lib, engine

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if name in ("pb200_ctx_create", "pb200_ctx_destroy", "pb200_ctx_set_stream", "pb200_last_error", "pb200_version"):
            return fn
        eng = self._engine

        def call(*args):
            cur = torch.cuda.current_stream(eng.device).cuda_stream
            if cur != eng._stream:
                self._lib.pb200_ctx_set_stream(eng.h, C.c_void_p(cur))
                eng._stream = cur
            return fn(*args)
        return call


class Engine:
    """One context = one device; work is enqueued on torch's current stream of that device (followed per call)."""

    def __init__(self, device=None):
        if not torch.cuda.is_available():
            raise RuntimeError("polara_b200 needs a CUDA device (sm_90); there is no CPU fallback")
        self.lib = _StreamFollowingLib(_abi.load(), self)
        self.device = torch.device("cuda", torch.cuda.current_device() if device is None else int(device))
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream(self.device).cuda_stream
        self._stream = stream
        handle = C.c_void_p()
        st = self.lib.pb200_ctx_create(self.device.index, C.c_void_p(stream), C.byref(handle))
        if st != _abi.OK:
            raise RuntimeError("pb200_ctx_create failed with status %d (an sm_90 GPU, H100, is required)" % st)
        self.h = handle
        self.score_kernel = "tc"       # the context's default; set_score_kernel keeps this copy current

    def close(self):
        if getattr(self, "h", None):
            self.lib.pb200_ctx_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---------------------------------------------------------------- helpers --
    def _check(self, st, where):
        try:
            _abi.check(self.h, st, where)
        except Exception as err:
            # a Python exception inside a reduce / bound hook cannot unwind through the C frames: it was parked and the
            # C call returned "hook failed"; surface the real cause
            cause = getattr(self, "_reduce_error", None)
            if cause is not None:
                self._reduce_error = None
                raise err from cause
            raise

    def empty(self, shape, dtype=torch.float32):
        return torch.empty(shape, dtype=dtype, device=self.device)

    def zeros(self, shape, dtype=torch.float32):
        return torch.zeros(shape, dtype=dtype, device=self.device)

    def upload(self, array, dtype=None):
        """numpy / host tensor -> device tensor (async on the context stream when pinned)."""
        if isinstance(array, torch.Tensor):
            t = array
        else:
            t = torch.from_numpy(np.ascontiguousarray(array))
        if dtype is not None and t.dtype != dtype:
            t = t.to(dtype)
        return t.to(self.device, non_blocking=True)

    def upload_csr(self, indptr, indices, values, shape):
        return DeviceCSR(self.upload(indptr, torch.int64), self.upload(indices, torch.int32),
                         self.upload(values, torch.float32), shape)

    def sync(self):
        self._check(self.lib.pb200_ctx_sync(self.h), "sync")

    def set_score_kernel(self, kind):
        code = {"simt": 0, "tc": 1}.get(kind, kind)
        self._check(self.lib.pb200_set_score_kernel(self.h, int(code)), "set_score_kernel")
        self.score_kernel = ("simt", "tc")[int(code)]

    @contextlib.contextmanager
    def score_kernel_scope(self, kind):
        """``kind`` in force inside the block (None: the current kind).  The engine is one per device and shared by every
        model, so the kind it had before is restored after the block, also when the block raises."""
        before = self.score_kernel
        if kind is None or kind == before:
            yield
            return
        self.set_score_kernel(kind)
        try:
            yield
        finally:
            self.set_score_kernel(before)

    def set_spmm_kernel(self, kind):
        kind = {"ldg": 0, "bulk": 1, "cpasync": 2, "window": 3, "window32": 4}.get(kind, kind)
        self._check(self.lib.pb200_set_spmm_kernel(self.h, int(kind)), "set_spmm_kernel")

    def set_prune(self, on):
        """norm-bound early termination of the fused scoring sweep (exact; on by default)."""
        self._check(self.lib.pb200_set_prune(self.h, int(bool(on))), "set_prune")

    def set_reduce_hook(self, reduce=None):
        """Install (or with None remove) the global-sum hook of the row-sharded build.  ``reduce(tensor)`` must sum the
        CUDA tensor in place over all ranks, ordered on the current stream (``torch.distributed.all_reduce``)."""
        if reduce is None:
            self._check(self.lib.pb200_set_reduce_hook(self.h, None, None), "set_reduce_hook")
            self._reduce_cb = None
            return
        dev = self.device
        dtypes = {0: (torch.float32, "<f4"), 1: (torch.float64, "<f8"), 2: (torch.int32, "<i4")}

        class _Span:                                   # raw device pointer -> torch tensor (zero copy)
            def __init__(self, p, count, typestr):
                self.__cuda_array_interface__ = {"shape": (int(count),), "typestr": typestr, "data": (int(p), False),
                                                 "version": 2}

        def hook(_user, p, count, dtype):
            try:
                tdtype, typestr = dtypes[int(dtype)]
                t = torch.as_tensor(_Span(p, count, typestr), device=dev)
                assert t.dtype == tdtype and t.data_ptr() == int(p)
                reduce(t)
                return 0
            except Exception as exc:                   # never unwind through the C frames
                self._reduce_error = exc
                return 1
        self._reduce_cb = _abi.REDUCE_FN(hook)         # keep the trampoline alive
        self._reduce_error = None
        self._check(self.lib.pb200_set_reduce_hook(self.h, C.cast(self._reduce_cb, C.c_void_p), None), "set_reduce_hook")

    def set_bound_hook(self, bound_max=None):
        """Install (or with None remove) the hook of item-sharded scoring (pb200_set_bound_hook): ``bound_max(tensor)`` must
        replace the float32 CUDA tensor of per-user lower bounds by its elementwise maximum over all ranks, ordered on the
        current stream (``torch.distributed.all_reduce(t, op=ReduceOp.MAX)``)."""
        if bound_max is None:
            self._check(self.lib.pb200_set_bound_hook(self.h, None, None), "set_bound_hook")
            self._bound_cb = None
            return
        dev = self.device

        class _Span:
            def __init__(self, p, count):
                self.__cuda_array_interface__ = {"shape": (int(count),), "typestr": "<f4", "data": (int(p), False), "version": 2}

        def hook(_user, p, count, dtype):
            try:
                assert int(dtype) == 0
                t = torch.as_tensor(_Span(p, count), device=dev)
                assert t.dtype == torch.float32 and t.data_ptr() == int(p)
                bound_max(t)
                return 0
            except Exception as exc:                   # never unwind through the C frames
                self._reduce_error = exc
                return 1
        self._bound_cb = _abi.REDUCE_FN(hook)          # keep the trampoline alive
        self._reduce_error = None
        self._check(self.lib.pb200_set_bound_hook(self.h, C.cast(self._bound_cb, C.c_void_p), None), "set_bound_hook")

    def stats(self):
        out = (C.c_uint64 * 8)()
        self._check(self.lib.pb200_get_stats(self.h, out), "get_stats")
        return [int(x) for x in out]

    # ------------------------------------------------------------------- ops ---
    def spmm(self, a: DeviceCSR, x, ell=None, out=None):
        """Y = A @ X ; X [n_cols x ldx] float32, uses the leading ``ell`` columns.  Y is [n_rows x round_up(ell, 32)],
        zero beyond column ``ell`` (padding columns are neither gathered nor accumulated)."""
        ell = x.shape[1] if ell is None else ell
        if out is None:
            out = self.empty((a.shape[0], round_up(ell, 32)))
        if a.n_panels > 1:
            view = a.view()
            st = self.lib.pb200_spmm_csr(self.h, C.byref(view), _p(x, _F32), x.stride(0), _p(out, _F32), out.stride(0), ell)
        else:
            st = self.lib.pb200_spmm(self.h, a.shape[0], a.shape[1], a.nnz, _p(a.indptr, _I64), _p(a.indices, _I32),
                                     _p(a.values, _F32), _p(x, _F32), x.stride(0), _p(out, _F32), out.stride(0), ell)
        self._check(st, "spmm")
        return out

    # L2 budget for the dense panel one column panel of a matrix gathers from (H100: 50 MB L2 in two partitions; data
    # read through both may be held twice, so well under half of it is planned for)
    PANEL_BYTES = 16 << 20

    def panel_cols_for(self, n_cols, ell):
        """columns per panel so that the gathered slice of X (panel_cols rows of min(ell,128) floats) stays in L2;
        returns n_cols when the whole operand fits (no blocking needed)."""
        row_bytes = 4 * min(round_up(max(int(ell), 1), 32), 128)
        if n_cols * row_bytes <= self.PANEL_BYTES * 5 // 4:
            return int(n_cols)
        cols = max(1024, self.PANEL_BYTES // row_bytes)
        n_panels = -(-n_cols // cols)
        return int(-(-n_cols // n_panels))           # equal panels

    def block_columns(self, a: DeviceCSR, panel_cols):
        """panel-major copy of ``a`` (pb200_csr_block_columns); returns ``a`` itself when one panel suffices."""
        panel_cols = int(panel_cols)
        n_panels = max(1, -(-a.shape[1] // panel_cols))
        if n_panels == 1 or a.n_panels > 1:
            return a
        b_indptr = self.empty((n_panels * a.shape[0] + 1,), torch.int64)
        b_indices = self.empty((a.nnz,), torch.int32)
        b_values = self.empty((a.nnz,), torch.float32)
        panel_ptr = (C.c_int64 * (n_panels + 1))()
        st = self.lib.pb200_csr_block_columns(self.h, a.shape[0], a.shape[1], a.nnz, _p(a.indptr, _I64), _p(a.indices, _I32),
                                              _p(a.values, _F32), panel_cols, n_panels, _p(b_indptr), _p(b_indices),
                                              _p(b_values), C.cast(panel_ptr, C.c_void_p))
        self._check(st, "csr_block_columns")
        return DeviceCSR(b_indptr, b_indices, b_values, a.shape, n_panels, panel_cols, panel_ptr)

    def coo_to_csr(self, rows, cols, vals, shape, drop_zeros=False, require_sorted_rows=False):
        """device ingest (pb200_coo_to_csr): ``rows`` / ``cols`` int64 CUDA tensors (1-d, any element stride -- e.g. the
        two columns of the [nnz x 2] index array of ``to_coo``), ``vals`` float32/float64 CUDA tensor or None (= ones).
        Returns a DeviceCSR with duplicates summed and sorted columns."""
        nnz = int(rows.shape[0])
        n_rows, n_cols = int(shape[0]), int(shape[1])
        if rows.dtype != _I64 or cols.dtype != _I64 or not rows.is_cuda or not cols.is_cuda:
            raise TypeError("coo_to_csr: rows / cols must be int64 CUDA tensors")
        if vals is not None and vals.dtype not in (_F32, _F64):
            raise TypeError("coo_to_csr: values must be float32 or float64")
        if vals is not None and vals.stride(0) != 1:
            vals = vals.contiguous()
        indptr = self.empty((n_rows + 1,), torch.int64)
        indices = self.empty((max(nnz, 1),), torch.int32)
        values = self.empty((max(nnz, 1),), torch.float32)
        out_nnz = C.c_int64(0)
        st = self.lib.pb200_coo_to_csr(self.h, n_rows, n_cols, nnz, C.c_void_p(rows.data_ptr()), rows.stride(0) if nnz else 1,
                                       C.c_void_p(cols.data_ptr()), cols.stride(0) if nnz else 1,
                                       C.c_void_p(vals.data_ptr()) if vals is not None else None,
                                       1 if (vals is not None and vals.dtype == _F64) else 0, int(bool(drop_zeros)),
                                       int(bool(require_sorted_rows)), _p(indptr), _p(indices), _p(values), C.byref(out_nnz))
        self._check(st, "coo_to_csr")
        n = int(out_nnz.value)
        return DeviceCSR(indptr, indices[:n], values[:n], (n_rows, n_cols))

    def coo_to_csr_runs(self, rows, cols, vals, shape, drop_zeros=False, require_sorted_rows=False):
        """``coo_to_csr`` (same CSR, same bits) plus ``(perm, run_ptr)`` (pb200_coo_to_csr_runs): ``perm`` int64 [nnz] maps
        sorted positions to input triplets, ``run_ptr`` int64 [csr.nnz + 1] bounds each stored entry's run of summed
        duplicates.  ``csr_values_from_table`` rewrites the values from them.  Returns ``(csr, perm, run_ptr)``."""
        nnz = int(rows.shape[0])
        n_rows, n_cols = int(shape[0]), int(shape[1])
        if rows.dtype != _I64 or cols.dtype != _I64 or not rows.is_cuda or not cols.is_cuda:
            raise TypeError("coo_to_csr_runs: rows / cols must be int64 CUDA tensors")
        if vals is not None and vals.dtype not in (_F32, _F64):
            raise TypeError("coo_to_csr_runs: values must be float32 or float64")
        if vals is not None and vals.stride(0) != 1:
            vals = vals.contiguous()
        indptr = self.empty((n_rows + 1,), torch.int64)
        indices = self.empty((max(nnz, 1),), torch.int32)
        values = self.empty((max(nnz, 1),), torch.float32)
        perm = self.empty((max(nnz, 1),), torch.int64)
        run_ptr = self.empty((nnz + 1,), torch.int64)
        out_nnz = C.c_int64(0)
        st = self.lib.pb200_coo_to_csr_runs(self.h, n_rows, n_cols, nnz, C.c_void_p(rows.data_ptr()),
                                            rows.stride(0) if nnz else 1, C.c_void_p(cols.data_ptr()),
                                            cols.stride(0) if nnz else 1,
                                            C.c_void_p(vals.data_ptr()) if vals is not None else None,
                                            1 if (vals is not None and vals.dtype == _F64) else 0, int(bool(drop_zeros)),
                                            int(bool(require_sorted_rows)), _p(indptr), _p(indices), _p(values),
                                            C.byref(out_nnz), _p(perm), _p(run_ptr))
        self._check(st, "coo_to_csr_runs")
        n = int(out_nnz.value)
        return DeviceCSR(indptr, indices[:n], values[:n], (n_rows, n_cols)), perm[:nnz], run_ptr[:n + 1]

    def csr_values_from_table(self, a: DeviceCSR, perm, run_ptr, levels, table):
        """In place: ``a.values`` <- the per-entry sums of ``table[levels]`` over the runs of ``coo_to_csr_runs``
        (pb200_csr_values_from_table), the bits a fresh ``coo_to_csr`` of the float32 weights ``table[levels]`` gives.
        ``levels`` int64 CUDA tensor [nnz input triplets], ``table`` float32 CUDA tensor [n_levels]."""
        if levels.dim() != 1 or levels.shape[0] != perm.shape[0]:
            raise ValueError("csr_values_from_table: one level per input triplet expected")
        if table.dim() != 1 or table.shape[0] < 1:
            raise ValueError("csr_values_from_table: the table must be a non-empty vector")
        if run_ptr.shape[0] != a.nnz + 1 or a.n_panels != 1:
            raise ValueError("csr_values_from_table: run bounds do not belong to this CSR")
        st = self.lib.pb200_csr_values_from_table(self.h, a.nnz, _p(run_ptr, _I64), _p(perm, _I64),
                                                  _p(levels.contiguous(), _I64), _p(table.contiguous(), _F32),
                                                  table.shape[0], _p(a.values, _F32))
        self._check(st, "csr_values_from_table")
        return a

    def rotate_factor(self, v, rot, out=None):
        """fp32(V R) zero padded to ``round_up(r, 32)`` columns (pb200_rotate_factor): ``v`` float64 CUDA tensor [n x K]
        (row stride >= K), ``rot`` float64 CUDA tensor [K x r], K, r <= 1024.  Returns the float32 [n x ld] tensor."""
        if v.dim() != 2 or rot.dim() != 2 or rot.shape[0] != v.shape[1]:
            raise ValueError("rotate_factor: expected V [n x K] and R [K x r]")
        n, k = v.shape
        r = rot.shape[1]
        if out is None:
            out = self.empty((n, round_up(r, 32)))
        st = self.lib.pb200_rotate_factor(self.h, n, k, r, _p(v, _F64), v.stride(0), _p(rot, _F64), rot.stride(0),
                                          _p(out, _F32), out.stride(0))
        self._check(st, "rotate_factor")
        return out

    def shift_i64(self, t, delta):
        """t += delta in place (int64 CUDA tensor): re-basing row pointers / user ids of a chunk."""
        st = self.lib.pb200_shift_i64(self.h, _p(t, _I64), t.numel(), int(delta))
        self._check(st, "shift_i64")
        return t

    def transpose(self, a: DeviceCSR):
        t = DeviceCSR(self.empty((a.shape[1] + 1,), torch.int64), self.empty((a.nnz,), torch.int32),
                      self.empty((a.nnz,), torch.float32), (a.shape[1], a.shape[0]))
        st = self.lib.pb200_csr_transpose(self.h, a.shape[0], a.shape[1], a.nnz, _p(a.indptr), _p(a.indices),
                                          _p(a.values, _F32), _p(t.indptr), _p(t.indices), _p(t.values))
        self._check(st, "csr_transpose")
        return t

    def rescale(self, a: DeviceCSR, row_scaling, col_scaling):
        st = self.lib.pb200_rescale(self.h, a.shape[0], a.shape[1], a.nnz, _p(a.indptr), _p(a.indices),
                                    _p(a.values, _F32), float(row_scaling), float(col_scaling))
        self._check(st, "rescale")

    def rsvd(self, a: DeviceCSR, at: DeviceCSR, rank, ell, max_iters=8, tol=1e-6, seed=1, want_u=False, vec_tol=0.0,
             item_factor=None, user_factor=None):
        """returns (V, sigma, U | None, iters); convergence details of the call are left in ``self.last_rsvd_info``:
        ``dict(iters, value_change, angle_bound, converged)`` (see pb200_rsvd_csr).

        ``item_factor`` / ``user_factor``: ``(K, K^T)`` pairs of DeviceCSR; with either the factorised operator is the
        matrix-free ``K_u^T A K_i`` (pb200_rsvd_factored), a missing side being the identity.  A factor whose gathered
        operand (its column count x ``ell`` floats) exceeds ``PANEL_BYTES`` is stored panel-major (``block_columns``)
        for the call, as the caller does for A and A^T."""
        ldv = round_up(rank, 32)
        v = self.zeros((a.shape[1], ldv))
        sigma = self.empty((rank,), torch.float64)
        u = self.zeros((a.shape[0], ldv)) if want_u else None
        info = (C.c_double * 8)()
        va, vt = a.view(), at.view()
        if item_factor is None and user_factor is None:
            st = self.lib.pb200_rsvd_csr(self.h, C.byref(va), C.byref(vt), rank, ell, max_iters, float(tol),
                                         float(vec_tol), int(seed), _p(v), ldv, _p(sigma), _p(u), ldv, info)
        else:
            keep, views = [], []
            for pair in (item_factor, user_factor):
                for k in (pair if pair is not None else (None, None)):
                    if k is None:
                        views.append(None)
                        continue
                    k = self.block_columns(k, self.panel_cols_for(k.shape[1], ell))
                    keep.append(k)                     # the views hold raw pointers into these
                    views.append(C.byref(k.view()))
            st = self.lib.pb200_rsvd_factored(self.h, C.byref(va), C.byref(vt), *views, rank, ell, max_iters,
                                              float(tol), float(vec_tol), int(seed), _p(v), ldv, _p(sigma), _p(u), ldv,
                                              info)
        self._check(st, "rsvd")
        self.last_rsvd_info = dict(iters=int(info[0]), value_change=float(info[1]), angle_bound=float(info[2]),
                                   converged=bool(info[3]))
        return v, sigma, u, int(info[0])

    def tall_svd(self, m, rank, want_vt=False):
        n, c = m.shape
        ldu = round_up(rank, 32)
        u = self.zeros((n, ldu))
        sigma = self.empty((rank,), torch.float64)
        vt = self.empty((rank, c)) if want_vt else None
        st = self.lib.pb200_tall_svd(self.h, _p(m, _F32), n, c, m.stride(0), rank, _p(sigma), _p(u), ldu, _p(vt))
        self._check(st, "tall_svd")
        return u, sigma, vt

    def score_topk(self, e, v, r, k, seen=None, item_offset=0, want_scores=False, m=None):
        m = e.shape[0] if m is None else m
        ids = self.empty((m, k), torch.int64)
        scores = self.empty((m, k), torch.float32) if want_scores else None
        sp, si = (seen if seen is not None else (None, None))
        st = self.lib.pb200_score_topk(self.h, _p(e, _F32), e.stride(0), _p(v, _F32), v.stride(0), m, v.shape[0], r,
                                       _p(sp, _I64), _p(si, _I32), k, item_offset, _p(ids), _p(scores))
        self._check(st, "score_topk")
        return (ids, scores) if want_scores else ids

    def last_score_kernel_ms(self):
        """duration of the last fused scoring kernel (CUDA events inside the library)."""
        return self.stats()[4] / 1000.0

    def score_topk_cands(self, e, v, r, k, seen=None, item_offset=0, m=None, m_alloc=None, bound_max=None):
        """candidate lists of ALL users against one item shard.  ``bound_max`` (see ``set_bound_hook``) shares the seed bounds
        between the shards for the duration of this call."""
        m = e.shape[0] if m is None else m
        m_alloc = m if m_alloc is None else m_alloc
        # {f32 score, i32 id} pairs; rows >= m (padding for the exchange) are empty lists
        cands = torch.empty((m_alloc, k, 2), dtype=torch.int32, device=self.device)
        if m_alloc > m:
            self._check(self.lib.pb200_fill_empty_cands(self.h, C.c_void_p(cands[m:].data_ptr()), (m_alloc - m) * k),
                        "fill_empty_cands")
        sp, si = (seen if seen is not None else (None, None))
        if bound_max is not None:
            self.set_bound_hook(bound_max)
        try:
            st = self.lib.pb200_score_topk_cands(self.h, _p(e, _F32), e.stride(0), _p(v, _F32), v.stride(0), m, v.shape[0], r,
                                                 _p(sp, _I64), _p(si, _I32), k, item_offset, _p(cands))
        finally:
            if bound_max is not None:
                self.set_bound_hook(None)
        self._check(st, "score_topk_cands")
        return cands

    def merge_cands(self, cands, parts, m, k, want_scores=False):
        ids = self.empty((m, k), torch.int64)
        scores = self.empty((m, k), torch.float32) if want_scores else None
        st = self.lib.pb200_merge_cands(self.h, _p(cands), parts, m, k, _p(ids), _p(scores))
        self._check(st, "merge_cands")
        return (ids, scores) if want_scores else ids

    def merge_cands_fill(self, cands, parts, part_rows, m, k, e, v, r, seen):
        """merge + seen-item fill-up for the rows this rank owns (pb200_merge_cands_fill).  ``cands`` [parts, part_rows, k, 2];
        ``e`` [>= m rows] embeddings of those rows, ``v`` the whole item factor matrix, ``seen`` = (indptr view starting at
        the first owned row, global indices)."""
        ids = self.empty((part_rows, k), torch.int64)
        st = self.lib.pb200_merge_cands_fill(self.h, _p(cands), parts, part_rows * k, m, k, _p(e, _F32), e.stride(0),
                                             _p(v, _F32), v.stride(0), r, v.shape[0], _p(seen[0], _I64), _p(seen[1], _I32),
                                             _p(ids), None)
        self._check(st, "merge_cands_fill")
        return ids

    def gather_dot(self, e, v, r, user_idx, item_idx):
        """scores of explicit (user, item) pairs: ``user_idx`` / ``item_idx`` int64 CUDA tensors of one shape; returns
        float32 scores of that shape (pb200_gather_dot)."""
        out = self.empty(tuple(user_idx.shape), torch.float32)
        st = self.lib.pb200_gather_dot(self.h, _p(e, _F32), e.stride(0), e.shape[0], _p(v, _F32), v.stride(0), v.shape[0], r,
                                       _p(user_idx.contiguous(), _I64), _p(item_idx.contiguous(), _I64), user_idx.numel(), _p(out))
        self._check(st, "gather_dot")
        return out

    def set_sampler_map_slots(self, slots):
        """shared-memory budget (8-byte slots per warp) of the sampler's position map (pb200_set_sampler_map_slots);
        users whose map does not fit run with it in global memory.  0 sends every user there."""
        self._check(self.lib.pb200_set_sampler_map_slots(self.h, int(slots)), "set_sampler_map_slots")

    def sampler_stats(self):
        """the last sampler call: dict(smem_users, global_users, global_slots, launches) (pb200_sampler_stats)."""
        out = (C.c_uint64 * 4)()
        self._check(self.lib.pb200_sampler_stats(self.h, out), "sampler_stats")
        return dict(smem_users=int(out[0]), global_users=int(out[1]), global_slots=int(out[2]), launches=int(out[3]))

    def _seeds(self, seeds):
        """uint32 seeds -> device (as the int32 tensor of the same bits)."""
        if isinstance(seeds, torch.Tensor):
            return seeds if seeds.dtype == _I32 and seeds.is_cuda else self.upload(seeds.view(torch.int32))
        return self.upload(np.ascontiguousarray(seeds, dtype=np.uint32).view(np.int32))

    def sample_unseen(self, excl_indptr, excl_indices, seeds, n_items, n_samples, out=None):
        """the reference's on-the-fly draw of unseen items (pb200_sample_unseen): ``excl_indptr`` int64 / ``excl_indices``
        int32 CUDA tensors (ordered exclusion lists), ``seeds`` uint32 per user.  Returns int64 [m x n_samples], or fills the
        first n_samples columns of ``out`` (an int64 CUDA view [m x >= n_samples] with unit column stride)."""
        m = int(excl_indptr.shape[0]) - 1
        if out is None:
            out = self.empty((m, int(n_samples)), torch.int64)
        sd = self._seeds(seeds)
        st = self.lib.pb200_sample_unseen(self.h, m, int(n_items), _p(excl_indptr, _I64), _p(excl_indices, _I32), _p(sd, _I32),
                                          int(n_samples), _p(out, _I64), out.stride(0) if out.dim() > 1 else int(n_samples))
        self._check(st, "sample_unseen")
        return out

    def sampled_topk(self, e, v, r, holdout_items, excl_indptr, excl_indices, seeds, n_samples, k, want_scores=False):
        """sampled evaluation fused (pb200_sampled_topk): top-k positions in ``[holdout | sampled]`` per user.
        ``holdout_items`` int64 CUDA [m x h]."""
        m = int(excl_indptr.shape[0]) - 1
        h = int(holdout_items.shape[1]) if holdout_items.dim() > 1 else 0
        hold = holdout_items.contiguous() if h else None          # an [m x 0] tensor has no usable strides
        pos = self.empty((m, int(k)), torch.int64)
        scores = self.empty((m, int(k)), torch.float32) if want_scores else None
        sd = self._seeds(seeds)
        st = self.lib.pb200_sampled_topk(self.h, _p(e, _F32), e.stride(0), _p(v, _F32), v.stride(0), m, v.shape[0], int(r),
                                         _p(hold, _I64), h, _p(excl_indptr, _I64), _p(excl_indices, _I32), _p(sd, _I32),
                                         int(n_samples), int(k), _p(pos), _p(scores))
        self._check(st, "sampled_topk")
        return (pos, scores) if want_scores else pos

    def sampled_topk_ranks(self, e, v, ranks, holdout_items, excl_indptr, excl_indices, seeds, n_samples, k,
                           want_scores=False):
        """``sampled_topk`` at every rank of ``ranks`` (strictly ascending) with one draw per user
        (pb200_sampled_topk_ranks): returns positions int64 ``[R, m, k]``, block j bit-equal to
        ``sampled_topk(e, v, ranks[j], ...)``."""
        m = int(excl_indptr.shape[0]) - 1
        h = int(holdout_items.shape[1]) if holdout_items.dim() > 1 else 0
        hold = holdout_items.contiguous() if h else None          # an [m x 0] tensor has no usable strides
        ranks = [int(r) for r in ranks]
        rk = (C.c_int * max(len(ranks), 1))(*ranks)
        pos = self.empty((len(ranks), m, int(k)), torch.int64)
        scores = self.empty((len(ranks), m, int(k)), torch.float32) if want_scores else None
        sd = self._seeds(seeds)
        st = self.lib.pb200_sampled_topk_ranks(self.h, _p(e, _F32), e.stride(0), _p(v, _F32), v.stride(0), m, v.shape[0],
                                               C.cast(rk, C.c_void_p), len(ranks), _p(hold, _I64), h, _p(excl_indptr, _I64),
                                               _p(excl_indices, _I32), _p(sd, _I32), int(n_samples), int(k), _p(pos),
                                               _p(scores))
        self._check(st, "sampled_topk_ranks")
        return (pos, scores) if want_scores else pos

    # columns of one build CTA's row panel of S (fp64 in shared memory: 64 KB, three CTAs per SM)
    COOC_PANEL_COLS = 8192

    def cooc_build(self, a: DeviceCSR, implicit=False, at=None):
        """item-to-item matrix S = A^T A with a zero diagonal, fp64 [n_items x lds] (pb200_cooc_build); ``implicit`` takes
        sign(a_ui).  Refuses with MemoryError, before allocating anything, when S and the build's scratch do not fit the
        device's free memory (``cooc_memory_check``).  Returns ``S`` (its first n_items columns are the matrix)."""
        m, n = a.shape
        panel_cols = min(n, self.COOC_PANEL_COLS)
        n_panels = -(-n // panel_cols)
        scratch = (0 if at is not None else a.nbytes() + 8 * n) + (a.nbytes() + 8 * n_panels * m if n_panels > 1 else 0) \
            + 32 * n
        cooc_memory_check(n, scratch, self.free_bytes())
        if at is None:
            at = self.transpose(a)
        a_blk = self.block_columns(a, panel_cols)
        lds = cooc_lds(n)
        s = self.empty((n, lds), torch.float64)
        va, vt = a_blk.view(), at.view()
        st = self.lib.pb200_cooc_build(self.h, C.byref(va), C.byref(vt), int(bool(implicit)), _p(s, _F64), lds)
        self._check(st, "cooc_build")
        return s

    def free_bytes(self):
        """free device memory in bytes: what the item-to-item builds check their allocations against."""
        return torch.cuda.mem_get_info(self.device)[0]

    # global scratch of the sparse item-to-item kernels: rows of n_items doubles for the item rows (build) and the users
    # (scoring) too long for a shared-memory table; the row count is capped by a byte budget and a row limit.  Scoring
    # gets the larger budget: each of its rows is one warp, and those warps are what keeps the HBM busy on long users.
    COOC_CSR_ACC_BYTES, COOC_CSR_ACC_ROWS = 256 << 20, 512        # build: one CTA of 256 threads per row
    I2I_CSR_ACC_BYTES, I2I_CSR_ACC_ROWS = 2 << 30, 2048           # scoring: one warp per row

    @staticmethod
    def _csr_acc_rows(n_items, budget, limit):
        return int(max(1, min(limit, budget // (8 * max(int(n_items), 1)))))

    def cooc_build_csr(self, a: DeviceCSR, implicit=False, at=None):
        """the item-to-item matrix of ``cooc_build`` as a DeviceCSR with float64 values (pb200_cooc_build_csr): sorted
        column ids, no diagonal, no stored zero, every entry bit-equal to the dense build's.  Two passes: the first counts
        the entries; ``cooc_csr_memory_check`` then refuses with MemoryError, before the rows are allocated, when they
        and the second pass's scratch do not fit the device's free memory.  The same check runs before the first pass
        on its scratch alone."""
        m, n = a.shape
        if a.n_panels > 1:
            raise ValueError("cooc_build_csr: `a` must be a plain CSR")
        rows = self._csr_acc_rows(n, self.COOC_CSR_ACC_BYTES, self.COOC_CSR_ACC_ROWS)
        scratch = rows * n * 8 + csr_sort_scratch_bytes(n)     # global rows (at most), schedule and sort buffers
        cooc_csr_memory_check(0, n, scratch + (0 if at is not None else a.nbytes() + 8 * n), self.free_bytes())
        if at is None:
            at = self.transpose(a)
        indptr = self.empty((n + 1,), torch.int64)
        total = C.c_int64(0)
        va, vt = a.view(), at.view()
        st = self.lib.pb200_cooc_build_csr(self.h, C.byref(va), C.byref(vt), int(bool(implicit)), rows, 0,
                                           _p(indptr, _I64), None, None, C.byref(total))
        self._check(st, "cooc_build_csr")
        nnz = int(total.value)
        try:
            # the first pass's scratch goes back to the device once its frees have run; indptr is already allocated:
            # it counts in the need and in what is free
            self.sync()
            cooc_csr_memory_check(nnz, n, scratch, self.free_bytes() + indptr.numel() * 8)
        except MemoryError:
            del indptr, at, va, vt                         # nothing of the build outlives the refusal
            raise
        indices = self.empty((nnz,), torch.int32)
        values = self.empty((nnz,), torch.float64)
        # with nnz == 0 both tensors are empty and their pointers NULL: the fill call then only returns
        st = self.lib.pb200_cooc_build_csr(self.h, C.byref(va), C.byref(vt), int(bool(implicit)), rows, 1,
                                           _p(indptr, _I64), _p(indices, _I32), _p(values, _F64), C.byref(total))
        self._check(st, "cooc_build_csr")
        return DeviceCSR(indptr, indices, values, (n, n))

    def i2i_topk_csr(self, s_csr: DeviceCSR, p: DeviceCSR, k, seen=None, implicit=False, want_scores=False):
        """``i2i_topk`` with S a float64 DeviceCSR (``cooc_build_csr``, or a caller's item x item matrix) through
        pb200_i2i_topk_csr: the same outputs, bit-equal to ``i2i_topk`` on the dense form of the same S.  Refuses with
        MemoryError, before allocating anything, when the outputs, the lists and one global row do not fit the device's
        free memory; the global rows take at most half of what is left (``I2I_CSR_ACC_BYTES`` at most)."""
        n = s_csr.shape[1]
        if s_csr.shape[0] != n or p.shape[1] != n:
            raise ValueError("i2i_topk_csr: S must be [n_items x n_items] and P [m x n_items]")
        m = p.shape[0]
        fixed = m * (8 + 8 * k * (3 if want_scores else 2)) + m * 2 * k * 16 + csr_sort_scratch_bytes(m)
        free = self.free_bytes()
        if fixed + 8 * n > free:
            raise MemoryError("item-to-item scoring: %d test users at k = %d need %d bytes of outputs and scratch plus "
                              "%d for one accumulator row, but only %d bytes of device memory are free"
                              % (m, k, fixed, 8 * n, free))
        rows = self._csr_acc_rows(n, min(self.I2I_CSR_ACC_BYTES, (free - fixed) // 2), self.I2I_CSR_ACC_ROWS)
        nnz = self.empty((m,), torch.int64)
        dense = self.empty((m, k), torch.int64)
        sparse = self.empty((m, k), torch.int64)
        scores = self.empty((m, k), torch.float64) if want_scores else None
        sp, si = (seen if seen is not None else (None, None))
        st = self.lib.pb200_i2i_topk_csr(self.h, n, _p(s_csr.indptr, _I64), _p(s_csr.indices, _I32),
                                         _p(s_csr.values, _F64), m, _p(p.indptr, _I64), _p(p.indices, _I32),
                                         _p(p.values, _F32), _p(sp, _I64), _p(si, _I32), int(bool(implicit)), int(k),
                                         rows, _p(nnz), _p(dense), _p(sparse), _p(scores))
        self._check(st, "i2i_topk_csr")
        return (nnz, dense, sparse, scores) if want_scores else (nnz, dense, sparse)

    def i2i_topk(self, s, n_items, p: DeviceCSR, k, seen=None, implicit=False, want_scores=False):
        """per test user the nonzero count of ``P S`` and its top-k lists under the dense and the sparse chunk rule
        (pb200_i2i_topk): returns ``(nnz int64 [m], dense int64 [m x k], sparse int64 [m x k])`` plus the fp64 scores of
        the dense lists with ``want_scores``."""
        m = p.shape[0]
        nnz = self.empty((m,), torch.int64)
        dense = self.empty((m, k), torch.int64)
        sparse = self.empty((m, k), torch.int64)
        scores = self.empty((m, k), torch.float64) if want_scores else None
        sp, si = (seen if seen is not None else (None, None))
        st = self.lib.pb200_i2i_topk(self.h, _p(s, _F64), s.stride(0), int(n_items), m, _p(p.indptr, _I64),
                                     _p(p.indices, _I32), _p(p.values, _F32), _p(sp, _I64), _p(si, _I32),
                                     int(bool(implicit)), int(k), _p(nnz), _p(dense), _p(sparse), _p(scores))
        self._check(st, "i2i_topk")
        return (nnz, dense, sparse, scores) if want_scores else (nnz, dense, sparse)

    def score_dense(self, e, v, r):
        m, n = e.shape[0], v.shape[0]
        s = self.empty((m, n))
        st = self.lib.pb200_score_dense(self.h, _p(e, _F32), e.stride(0), _p(v, _F32), v.stride(0), m, n, r, _p(s), n)
        self._check(st, "score_dense")
        return s

    def topk_dense(self, scores, k, seen=None, want_scores=False):
        """top-k of a dense CUDA score block [m x n] (float32 / float64), optional fused seen handling (pb200_topk_dense)."""
        if scores.dtype not in (_F32, _F64):
            raise TypeError("topk_dense: scores must be float32 or float64")
        m, n = scores.shape
        ids = self.empty((m, k), torch.int64)
        out = self.empty((m, k), scores.dtype) if want_scores else None
        sp, si = (seen if seen is not None else (None, None))
        st = self.lib.pb200_topk_dense(self.h, _p(scores), 1 if scores.dtype == _F64 else 0, scores.stride(0), m, n,
                                       _p(sp, _I64), _p(si, _I32), int(k), _p(ids), _p(out))
        self._check(st, "topk_dense")
        return (ids, out) if want_scores else ids

    def downvote_dense(self, scores, rows, cols):
        """in place: push the scores at (rows, cols) below the block minimum, order preserved (pb200_downvote_dense)."""
        m, n = scores.shape
        st = self.lib.pb200_downvote_dense(self.h, _p(scores), 1 if scores.dtype == _F64 else 0, scores.stride(0), m, n,
                                           _p(rows, _I64), _p(cols, _I64), int(rows.shape[0]))
        self._check(st, "downvote_dense")
        return scores

    def coo_group(self, key, n_keys, a, b, val):
        nnz = key.shape[0]
        seg = self.empty((n_keys + 1,), torch.int64)
        ao, bo = self.empty((nnz,), torch.int32), self.empty((nnz,), torch.int32)
        vo = self.empty((nnz,), torch.float32)
        st = self.lib.pb200_coo_group(self.h, nnz, n_keys, _p(key, _I32), _p(a, _I32), _p(b, _I32), _p(val, _F32), _p(seg), _p(ao), _p(bo), _p(vo))
        self._check(st, "coo_group")
        return seg, ao, bo, vo

    def ttm(self, n0, seg, i1, i2, val, u, ru, w, rw):
        """out[i0, x*rw + y] = sum_{nnz in row i0} val * u[i1, x] * w[i2, y]."""
        ldo = round_up(ru * rw, 4)
        out = self.empty((n0, ldo))
        st = self.lib.pb200_ttm(self.h, n0, i1.shape[0], _p(seg, _I64), _p(i1, _I32), _p(i2, _I32), _p(val, _F32), _p(u, _F32), ru, u.stride(0),
                                _p(w, _F32), rw, w.stride(0), _p(out), ldo)
        self._check(st, "ttm")
        return out

    def ttm_reduce(self, n_seg, seg, ia, ib, val, a, ra, b, rb):
        out = self.empty((n_seg, ra * rb))
        st = self.lib.pb200_ttm_reduce(self.h, n_seg, ia.shape[0], _p(seg, _I64), _p(ia, _I32), _p(ib, _I32), _p(val, _F32), _p(a, _F32), ra,
                                       a.stride(0), _p(b, _F32), rb, b.stride(0), _p(out), ra * rb)
        self._check(st, "ttm_reduce")
        return out


def cooc_lds(n_items):
    """row stride of the dense item-to-item matrix: rows start on 128-byte boundaries."""
    return round_up(int(n_items), 16)


def cooc_memory_check(n_items, scratch_bytes, free_bytes):
    """Raises MemoryError when the dense fp64 item-to-item matrix of ``n_items`` items plus ``scratch_bytes`` exceeds
    ``free_bytes`` (the device's free memory); larger catalogues take the sparse form (``cooc_build_csr``)."""
    need_s = int(n_items) * cooc_lds(n_items) * 8
    need = need_s + int(scratch_bytes)
    if need > int(free_bytes):
        raise MemoryError("item-to-item model: the dense item x item matrix of %d items takes %d bytes (plus %d bytes of "
                          "scratch, %d in all), but only %d bytes of device memory are free"
                          % (int(n_items), need_s, int(scratch_bytes), need, int(free_bytes)))
    return need


def csr_sort_scratch_bytes(count):
    """scratch of the sparse item-to-item kernels' longest-first schedule over ``count`` rows or users: work, order and
    the radix sort's key and value buffers (about 48 bytes each), with a fixed margin for the sort's and scan's
    temporary storage."""
    return 64 * int(count) + (16 << 20)


def cooc_csr_bytes(nnz, n_items):
    """bytes of the item-to-item matrix as an fp64 CSR: int64 row offsets, int32 column ids, fp64 values."""
    return 8 * (int(n_items) + 1) + 12 * int(nnz)


def cooc_csr_memory_check(nnz, n_items, scratch_bytes, free_bytes):
    """Raises MemoryError when the sparse fp64 item-to-item matrix of ``n_items`` items with ``nnz`` stored entries plus
    ``scratch_bytes`` exceeds ``free_bytes`` (the device's free memory)."""
    need_s = cooc_csr_bytes(nnz, n_items)
    need = need_s + int(scratch_bytes)
    if need > int(free_bytes):
        raise MemoryError("item-to-item model: the sparse item x item matrix of %d items with %d stored entries takes %d "
                          "bytes (plus %d bytes of scratch, %d in all), but only %d bytes of device memory are free"
                          % (int(n_items), int(nnz), need_s, int(scratch_bytes), need, int(free_bytes)))
    return need


_ENGINES = {}


def get_engine(device=None):
    """Process-wide engine per device (created on first use)."""
    if not torch.cuda.is_available():
        raise RuntimeError("polara_b200 needs a CUDA device (sm_90); there is no CPU fallback")
    idx = torch.cuda.current_device() if device is None else int(device)
    eng = _ENGINES.get(idx)
    if eng is None:
        eng = _ENGINES[idx] = Engine(idx)
    return eng
