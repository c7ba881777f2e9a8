"""GPU (H100, sm_90a) drop-ins for the reference's SVDModel / ScaledSVD / CoffeeModel hot path.

``build()`` and ``get_recommendations()`` run entirely on the device through the C-ABI
(:mod:`polara_b200.engine`); host code only converts the data model's COO arrays to CSR
and moves buffers.  There is no CPU fallback: without the CUDA library or an sm_90
device every call raises.

Two families of classes share the device logic (mixins below):

* ``B200SVDModel`` / ``B200ScaledSVD`` / ``B200CoffeeModel`` -- stand-alone, built on the
  mirror base in :mod:`polara_b200.host` (works without the reference installed);
* :func:`dropin` -- the same mixins grafted onto the *real* ``polara`` classes when that
  package is importable, so that ``polara.evaluation`` pipelines keep working unchanged.

The HybridSVD, item-to-item, SimilarityAggregation and item cold-start models follow the same pattern
(``dropin_hybrid``, ``dropin_i2i``, ``dropin_similarity``, ``dropin_coldstart``).
"""
from __future__ import annotations

import time

import numpy as np
import torch

from . import host
from .engine import DeviceCSR, get_engine, round_up

__all__ = ["B200SVDModel", "B200ScaledSVD", "B200HybridSVD", "B200ScaledHybridSVD", "B200CoffeeModel",
           "B200CooccurrenceModel", "B200SimilarityAggregation", "B200SVDModelItemColdStart",
           "B200ScaledSVDItemColdStart", "B200HybridSVDItemColdStart", "B200ScaledHybridSVDItemColdStart", "dropin",
           "dropin_coldstart", "dropin_hybrid", "dropin_i2i", "dropin_similarity", "default_ell"]


def default_ell(rank, oversample=None):
    """Subspace width of the randomized range finder: rank + max(22, rank/2), rounded to 32."""
    p = max(22, rank // 2) if oversample is None else oversample
    return min(1024, round_up(rank + p, 32))


def _pinned(arr):
    t = torch.from_numpy(np.ascontiguousarray(arr))
    try:
        return t.pin_memory()
    except RuntimeError:
        return t


def _as_index_array(x):
    """index arrays cross PCIe as int64 (what ``to_coo`` / ``test_to_coo`` produce: np.intp, data.py:815,849)."""
    x = np.asarray(x)
    return x if x.dtype == np.int64 else x.astype(np.int64)


def _as_value_array(x):
    x = np.asarray(x)
    return x if x.dtype in (np.float32, np.float64) else x.astype(np.float64)


class _DeviceModelMixin:
    """State shared by the device models: engine handle and cached device buffers."""

    _engine = None
    score_kernel = None          # None = the engine's current kind; 'simt' | 'tc'
    last_timings = None

    @property
    def engine(self):
        if self._engine is None:
            self._engine = get_engine()
        return self._engine

    @property
    def recommendations(self):
        """models.py:100-108, plus: on an item-sharded model ``get_recommendations()`` returns the lists of the users this
        rank owns; the cached ``recommendations`` (what ``evaluate()`` consumes, aligned with the holdout rows) are the
        lists of ALL users, all-gathered once."""
        if self._recommendations is None:
            if not self._is_ready:
                if self.verbose:
                    print("{} model is not ready. Rebuilding.".format(self.method))
                self.build()
            recs = self.get_recommendations()
            shard = getattr(self, "shard", None)
            if shard is not None and shard.world > 1:
                from .dist import gather_lists
                recs = gather_lists(recs, shard, None, self.engine.device)      # user count = sum of the ranks' shares
            self._recommendations = recs
        return self._recommendations

    def _device_factor(self, key, width_multiple=32):
        """Device copy [n x ld] (zero padded to a multiple of 32 columns) of the numpy factor
        ``self.factors[key]``; re-uploaded whenever the host array object changes (rank
        truncation, models.py:819-832, replaces the array by a view)."""
        host_arr = self.factors[key]
        cache = self.__dict__.setdefault("_dev_cache", {})
        hit = cache.get(key)
        if hit is not None and hit[0] is host_arr:
            return hit[1]
        r = host_arr.shape[1]
        ld = round_up(r, width_multiple)
        buf = np.zeros((host_arr.shape[0], ld), dtype=np.float32)
        buf[:, :r] = host_arr
        dev = self.engine.upload(buf)
        cache[key] = (host_arr, dev)
        return dev

    def _remember_device_factor(self, key, host_arr, dev):
        self.__dict__.setdefault("_dev_cache", {})[key] = (host_arr, dev)

    # ----- test data -> device CSR --------------------------------------------------
    def _test_csr_device(self, test_data, shape, values=None, stream_arrays=None, sorted_users=False):
        """Device CSR of the test matrix P (zero feedback dropped, models.py:197-201; duplicates summed, models.py:208-210)
        and the (indptr, indices) pair of the *seen* pattern (ALL triplets, models.py:191-196,211), built on the device
        from the triplets of ``_get_test_data`` (pb200_coo_to_csr).  ``values`` (CoFFee: per-triplet weights, the feedback
        there is an index, never "zero feedback") replaces the feedback as matrix values; nothing is dropped then."""
        eng = self.engine
        n_users, n_items = int(shape[0]), int(shape[1])
        if stream_arrays is None:
            user, item, fdbk = test_data
        if stream_arrays is not None:
            u_d, i_d, f_d, w_d = stream_arrays
        else:
            u_d, i_d = eng.upload(_as_index_array(user)), eng.upload(_as_index_array(item))
            f_d = None if values is not None else eng.upload(_as_value_array(fdbk))
            w_d = None if values is None else eng.upload(_as_value_array(values))
        if w_d is None:
            p = eng.coo_to_csr(u_d, i_d, f_d, (n_users, n_items), drop_zeros=True, require_sorted_rows=sorted_users)
        else:
            p = eng.coo_to_csr(u_d, i_d, w_d, (n_users, n_items), drop_zeros=False)
        if p.nnz == int(u_d.shape[0]):
            seen = (p.indptr, p.indices)          # nothing dropped, nothing merged: same pattern
        else:
            s = eng.coo_to_csr(u_d, i_d, None, (n_users, n_items), drop_zeros=False)
            seen = (s.indptr, s.indices)
        return p, seen

    def _item_projector_device(self, v_dev):
        """HybridSVD scores with two item-side matrices, ``scores = P . vr . vl^T`` (hybrid/models.py:390-394:
        ``<itemid>_projector_right`` folds the history in, ``<itemid>_projector_left`` scores); a model that carries them
        in ``factors`` is scored the same way, everything else with the item factors on both sides."""
        itemid = self.data.fields.itemid
        vl = self.factors.get("%s_projector_left" % itemid)
        vr = self.factors.get("%s_projector_right" % itemid)
        if vl is None or vr is None:
            return v_dev, v_dev
        if getattr(self, "shard", None) is not None:
            raise NotImplementedError("item projectors on an item-sharded model")
        return self._device_factor("%s_projector_right" % itemid), self._device_factor("%s_projector_left" % itemid)

    def _checked_test_input(self, read):
        """``read()``, a reader of the test data that returns their shape second, between the checks the reference makes
        around it: data integrity before, ``topk`` against the item count after (np.argpartition would raise,
        models.py:490)."""
        if self.verify_integrity and hasattr(self, "verify_data_integrity"):
            self.verify_data_integrity()
        test_input = read()
        if self.topk > test_input[1][1]:
            raise ValueError("topk exceeds the number of items")
        return test_input

    def _rank_lists(self, p_dev: DeviceCSR, seen_dev, v_fold, v_score, ranks):
        """E = P v_fold once, at the padded width of the largest of the ascending ``ranks`` (the faster, unpredicated SpMM
        variant), then the fused scoring kernel against ``v_score``: one int64 [m x topk] device tensor per rank."""
        eng = self.engine
        e = eng.spmm(p_dev, v_fold, ell=round_up(ranks[-1], 32))
        seen = seen_dev if self.filter_seen else None
        return [eng.score_topk(e, v_score, r, self.topk, seen=seen) for r in ranks]

    def _score(self, p_dev: DeviceCSR, seen_dev, v_dev, rank):
        v_fold, v_dev = self._item_projector_device(v_dev)
        shard = getattr(self, "shard", None)
        if shard is None:
            return self._rank_lists(p_dev, seen_dev, v_fold, v_dev, [rank])[0]
        # item-factor sharding: returns the lists of the user range this rank owns
        from .dist import sharded_topk
        eng = self.engine
        e = eng.spmm(p_dev, v_fold, ell=v_fold.shape[1])
        ids = sharded_topk(eng, e, v_dev, rank, self.topk, seen_dev if self.filter_seen else None, shard, p_dev.shape[0])
        lo, hi = shard.user_range(p_dev.shape[0])
        return ids[: hi - lo]


class _SVDDeviceMixin(_DeviceModelMixin):
    """Device implementation of SVDModel.build / get_recommendations
    (polara/recommender/models.py:835-861, 391-405)."""

    oversample = None        # subspace width = rank + oversample (None -> default_ell)
    power_iters = 12         # cap on subspace iterations
    tol = 1e-6               # stop when the leading Ritz values move less than this (relative) ...
    vec_tol = 1e-3           # ... and the leading-rank subspaces of two successive iterates are this close (sine bound)
    rsvd_seed = 1

    def _training_csr_device(self):
        data = self.data
        fast = getattr(data, "train_csr", None)
        if fast is not None:
            indptr, indices, values, shape = fast
        else:
            # the triplets of RecommenderData.to_coo go to the device as they are; the CSR is built there
            idx, val, shape = data.to_coo(tensor_mode=False, feedback_threshold=self.feedback_threshold)
            idx = _as_index_array(idx)
            val = _as_value_array(val)
            self._n_train_users = int(shape[0])
            rows = self._build_rows(shape[0])
            if rows is not None:
                # row-sharded build: this rank ingests only its block of user rows (re-based)
                keep = (idx[:, 0] >= rows[0]) & (idx[:, 0] < rows[1])
                idx = idx[keep] - np.array([rows[0], 0], dtype=np.int64)
                val = val[keep]
                shape = (rows[1] - rows[0], shape[1])
            eng = self.engine
            idx_d = eng.upload(np.ascontiguousarray(idx))
            a = eng.coo_to_csr(idx_d[:, 0], idx_d[:, 1], eng.upload(val), shape)
            return self._scaled(a)
        self._n_train_users = int(shape[0])
        rows = self._build_rows(shape[0])
        if rows is not None:
            # row-sharded build: this rank keeps (and copies to its GPU) only its block of user rows
            indptr, indices, values, shape = csr_row_block(indptr, indices, values, shape, rows[0], rows[1])
        a = self.engine.upload_csr(indptr, indices, values, shape)
        return self._scaled(a)

    def _scaled(self, a):
        row_s = getattr(self, "row_scaling", 1)
        col_s = getattr(self, "col_scaling", 1) if hasattr(self, "_col_scaling") else 1
        if hasattr(self, "_col_scaling"):
            self.engine.rescale(a, row_s, col_s)      # ScaledMatrixMixin, models.py:891-895
        return a

    def _build_rows(self, n_users):
        """user rows this rank factorises when the build is sharded (``self.shard`` set, world > 1), else None."""
        shard = getattr(self, "shard", None)
        if shard is None or shard.world <= 1 or not self.shard_build:
            return None
        return shard.user_range(n_users)

    def build(self, operator=None, return_factors="vh"):
        """models.py:835-855.  ``operator`` (``svd_matrix = operator``, models.py:836-837): an EXPLICIT sparse matrix of the
        training matrix's shape is factorised in its place -- what HybridSVD passes with ``precompute_auxiliary_matrix``
        (``L_K^T A L_S`` formed on the host, hybrid/models.py:364-370).  The matrix-free ``LinearOperator`` form wraps CHOLMOD
        solves on the host (hybrid/models.py:372-388) and has no device counterpart: NotImplementedError, as before."""
        op_csr = None
        if operator is not None:
            import scipy.sparse as sps
            if not sps.issparse(operator):
                raise NotImplementedError("only an explicit sparse matrix is accepted as `operator` on the device path "
                                          "(HybridSVD: set precompute_auxiliary_matrix = True); a LinearOperator is not")
            if self._build_rows(1) is not None:
                raise NotImplementedError("row-sharded build of an explicit operator")
            op_csr = sps.csr_matrix(operator)
            op_csr.sum_duplicates()
            op_csr.sort_indices()
        eng = self.engine
        sharded = self._build_rows(1) is not None
        if sharded:
            import torch.distributed as dist
            eng.set_reduce_hook(dist.all_reduce)       # sums Gram matrices / A^T W panels / column counts over ranks
        try:
            self._build_factors(eng, return_factors, sharded, op_csr)
        finally:
            if sharded:
                eng.set_reduce_hook(None)

    def _build_factors(self, eng, return_factors, sharded, op_csr=None, a=None, item_factor=None, user_factor=None):
        """``a``: the training matrix already on the device; ``item_factor`` / ``user_factor``: ``(K, K^T)`` DeviceCSR pairs
        of a factored operator ``K_u^T A K_i`` (Engine.rsvd)."""
        t0 = time.perf_counter()
        if a is None and op_csr is None:
            a = self._training_csr_device()
        elif a is None:
            a = eng.upload_csr(op_csr.indptr.astype(np.int64), op_csr.indices.astype(np.int32),
                               op_csr.data.astype(np.float32), op_csr.shape)
            self._n_train_users = op_csr.shape[0]
        at = eng.transpose(a)
        rank = self.rank
        ell = default_ell(rank, self.oversample)
        ell = min(ell, round_up(min(a.shape), 32)) if min(a.shape) >= 32 else 32
        # panel-major copies where the dense operand of a product would not stay L2-resident (A^T W gathers user rows:
        # 1e6 x 96 floats = 384 MB at C2); format conversion, part of the preparation like the transpose
        at = eng.block_columns(at, eng.panel_cols_for(at.shape[1], ell))
        a = eng.block_columns(a, eng.panel_cols_for(a.shape[1], ell))
        want_u = return_factors is True
        eng.sync()
        t1 = time.perf_counter()
        v, sigma, u, iters = eng.rsvd(a, at, rank, ell, max_iters=self.power_iters, tol=self.tol, vec_tol=self.vec_tol,
                                      seed=self.rsvd_seed, want_u=want_u, item_factor=item_factor,
                                      user_factor=user_factor)
        eng.sync()
        info = dict(eng.last_rsvd_info)
        if not info["converged"]:
            import warnings
            warnings.warn("%s: subspace iteration stopped at the cap of %d iterations -- leading Ritz values still move by "
                          "%.1e (tol %.1e), successive-subspace sine bound %.1e (tol %.1e).  The factors are the best "
                          "rank-%d subspace found, not a converged one (flat spectrum at the cut?); raise power_iters or "
                          "oversample." % (self.method, self.power_iters, info["value_change"], self.tol,
                                           info["angle_bound"], self.vec_tol, rank), RuntimeWarning, stacklevel=3)
        if sharded and u is not None:
            u = self._gather_user_rows(u)
        t2 = time.perf_counter()
        if self.training_time is not None:
            self.training_time.append(t2 - t1)       # what track_time covers, models.py:843
        if self.verbose:
            print("{} training time: {:.3f}s".format(self.method, t2 - t1))
        f = self.data.fields
        v_host = v[:, :rank].cpu().numpy().astype(np.float64)
        self.factors[f.userid] = None if u is None else u[:, :rank].cpu().numpy().astype(np.float64)
        self.factors[f.itemid] = v_host
        self.factors["singular_values"] = sigma.cpu().numpy()
        self._remember_device_factor(f.itemid, v_host, v)
        self.last_timings = dict(prepare_s=t1 - t0, rsvd_s=t2 - t1, subspace_iters=iters, ell=ell,
                                 panels=(a.n_panels, at.n_panels), converged=info["converged"],
                                 value_change=info["value_change"], angle_bound=info["angle_bound"])

    shard_build = True       # with ``self.shard`` set (world > 1) factorise row blocks in parallel (SURVEY.md 8e)

    def _gather_user_rows(self, u_local):
        """assemble the user factors from the row blocks of all ranks (one broadcast per rank)."""
        import torch.distributed as dist
        shard = self.shard
        n_users = self._n_train_users
        full = torch.empty((n_users, u_local.shape[1]), dtype=u_local.dtype, device=u_local.device)
        lo, hi = shard.user_range(n_users)
        full[lo:hi].copy_(u_local)
        c = shard.user_chunk(n_users)
        for src in range(shard.world):
            a, b = min(n_users, src * c), min(n_users, (src + 1) * c)
            if b > a:
                dist.broadcast(full[a:b], src=src)
        return full

    stream_chunks = None     # user chunks of a streamed scoring call (H2D of chunk i+1 overlaps scoring of chunk i);
                             # None = stream_schedule(), an int = that many equal chunks

    def get_recommendations(self):
        rows, shape, is_csr, streamable = self._checked_test_input(self._test_input)
        itemid = self.data.fields.itemid
        rank = self.factors[itemid].shape[1]
        with self.engine.score_kernel_scope(self.score_kernel):
            if getattr(self, "shard", None) is None:
                bounds = (streamable and self._stream_bounds(shape[0])) or [0, shape[0]]
                return self._chunked_lists(rows, shape, is_csr, bounds, [rank])[0]
            if is_csr and isinstance(rows[0], torch.Tensor):
                return self._sharded_recommendations(*rows, shape)
            if is_csr:
                p_dev = self.engine.upload_csr(*rows, shape[:2])
                seen_dev = (p_dev.indptr, p_dev.indices)
            else:
                p_dev, seen_dev = self._test_csr_device(rows, shape)
            return self._score(p_dev, seen_dev, self._device_factor(itemid), rank).cpu().numpy()

    def _test_input(self):
        """``(rows, shape, is_csr, streamable)`` of a scoring call: ``rows`` is the ``(indptr, indices, values)`` of
        ``data.test_csr`` when set, else the user-sorted ``(user, item, feedback)`` of ``_big_test_triplets()`` or else of
        ``_get_test_data()``.  ``streamable``: a torch CSR in host memory or the triplets of a large test set."""
        fast = getattr(self.data, "test_csr", None)
        if fast is not None:
            rows, shape = fast
            return rows, shape, True, isinstance(rows[0], torch.Tensor)
        big = self._big_test_triplets()
        if big is not None:
            return big[0], big[1], False, True
        test_data, shape, _ = self._get_test_data()
        return test_data, shape, False, False

    def _stream_bounds(self, m):
        """User-chunk bounds of a streamed scoring call over ``m`` test users, or None when there are too few to stream.
        The bounds fix the last bits of the result: SpMM windows are counted from each launch's first nnz (DESIGN.md
        section 4), so E, and with it a near-tied list, depends on where the rows are cut."""
        if m < 4 * 65536:
            return None
        if self.stream_chunks is None:
            sms = torch.cuda.get_device_properties(self.engine.device).multi_processor_count
            return stream_schedule(m, sms * 128)
        n_chunks = max(1, int(self.stream_chunks))
        return [m * c // n_chunks for c in range(n_chunks + 1)]

    def _big_test_triplets(self):
        """Large test sets (those that are streamed, ``_stream_bounds``) skip the host-side passes of ``_get_test_data``
        (models.py:227-257: np.diff over all triplets for the sortedness assert and the gap test -- four passes over 1e8
        int64 cost more than the whole device path).  The same facts are established differently: the ingest kernel checks
        the order of every chunk on the device (and sorts if it has to), and users that start at 0 and end at
        n_test_users - 1 leave no room for a gap because ``get_test_shape`` counts the distinct test users
        (data.py:865-884).  Anything else returns None and takes the reference's path."""
        if getattr(self, "shard", None) is not None:
            return None
        data = self.data
        shape = data.get_test_shape(tensor_mode=False)
        if self._stream_bounds(shape[0]) is None:
            return None
        threshold = None if data.warm_start else self.feedback_threshold
        user, item, fdbk = data.test_to_coo(tensor_mode=False, feedback_threshold=threshold)
        if len(user) == 0 or int(user[0]) != 0 or int(user[-1]) != shape[0] - 1:
            return None
        return (user, item, fdbk), shape

    def _sharded_recommendations(self, indptr, indices, values, shape):
        """Item-sharded scoring from a pinned host CSR that every rank holds: each rank copies only ITS slice of the rows
        over PCIe, the slices are exchanged GPU-to-GPU (one broadcast per rank over NVLink) so that every GPU ends up with
        the whole test matrix (needed for the user embeddings and the seen lists), then SpMM + fused scoring on the own
        item shard + all-to-all + merge.  Returns the lists of the user range this rank owns."""
        import torch.distributed as dist
        eng, shard = self.engine, self.shard
        m, n_items = shape[0], shape[1]
        rank_r = self.factors[self.data.fields.itemid].shape[1]
        v_dev = self._device_factor(self.data.fields.itemid)
        self._item_projector_device(v_dev)                    # raises for a model that carries item projectors
        indptr64 = indptr if indptr.dtype == torch.int64 else indptr.to(torch.int64)
        world = shard.world
        chunk_u = shard.user_chunk(m)
        row_bounds = [min(m, c * chunk_u) for c in range(world + 1)]       # the user ranges the ranks own (ItemShard)
        nnz_bounds = [int(indptr64[b]) for b in row_bounds]
        nnz = nnz_bounds[-1]
        prof = getattr(self, "profile_phases", False)
        tp = [time.perf_counter()]

        def mark():
            if prof:
                torch.cuda.synchronize()
                tp.append(time.perf_counter())
        ip_dev = indptr64.to(eng.device, non_blocking=True)
        ix_dev = torch.empty(nnz, dtype=torch.int32, device=eng.device)
        lo, hi = nnz_bounds[shard.rank], nnz_bounds[shard.rank + 1]
        ix_dev[lo:hi].copy_(indices[lo:hi], non_blocking=True)
        vl_blk = values[lo:hi].to(eng.device, non_blocking=True)        # values are needed for the own row block only
        mark()
        for src in range(world):
            a, b = nnz_bounds[src], nnz_bounds[src + 1]
            if b > a:
                dist.broadcast(ix_dev[a:b], src=src)                     # the seen lists of ALL users are needed everywhere
        from .dist import gather_embeddings, sharded_topk
        mark()
        # user embeddings: every rank multiplies its block of rows, the blocks are all-gathered (SURVEY.md 8e)
        r_lo, r_hi = row_bounds[shard.rank], row_bounds[shard.rank + 1]
        ip_blk = ip_dev[r_lo:r_hi + 1].clone()
        eng.shift_i64(ip_blk, -lo)
        p_block = DeviceCSR(ip_blk, ix_dev[lo:hi], vl_blk if vl_blk.dtype == torch.float32 else vl_blk.to(torch.float32),
                            (r_hi - r_lo, n_items))
        e = gather_embeddings(eng, p_block, v_dev, shard, m)
        seen = (ip_dev, ix_dev) if self.filter_seen else None
        ids = sharded_topk(eng, e, v_dev, rank_r, self.topk, seen, shard, m)
        mark()
        u_lo, u_hi = shard.user_range(m)
        out_t = torch.empty((u_hi - u_lo, self.topk), dtype=torch.int64, pin_memory=True)
        out_t.copy_(ids[: u_hi - u_lo], non_blocking=True)
        torch.cuda.current_stream(eng.device).synchronize()
        out = out_t.numpy()
        mark()
        if prof:
            self.last_score_timings = dict(zip(("h2d_s", "assemble_s", "score_s", "d2h_s"), np.diff(tp).round(4)))
        return out

    def _chunked_lists(self, rows, shape, is_csr, bounds, ranks):
        """Host test rows -> one int64 [m x topk] array of lists per rank of the ascending ``ranks``, scored in the user
        chunks ``bounds``: the H2D copy of chunk i+1 (side stream) overlaps ingest + SpMM + fused scoring of chunk i
        (context stream); the lists go back into one pinned buffer on a third stream.  One chunk has nothing to overlap and
        runs in order on the context stream (unless ``profile_phases`` wants its events).  ``rows``: a host CSR
        (``is_csr``; numpy or torch) or the user-sorted ``(user, item, feedback)`` arrays of ``test_to_coo``, converted
        to CSR on the device chunk by chunk (pb200_coo_to_csr)."""
        t_entry = time.perf_counter()
        eng = self.engine
        m, n_items = shape[0], shape[1]
        v_fold, v_score = self._item_projector_device(self._device_factor(self.data.fields.itemid))
        n_chunks = len(bounds) - 1
        prof = [] if getattr(self, "profile_phases", False) else None
        if is_csr:
            indptr, indices, values = (x if isinstance(x, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(x))
                                       for x in rows)
            indptr64 = indptr if indptr.dtype == torch.int64 else indptr.to(torch.int64)
            host = (indices, values)
        else:
            user, item, fdbk = (np.asarray(x) for x in rows)
            host = tuple(torch.from_numpy(x) for x in (_as_index_array(user), _as_index_array(item), _as_value_array(fdbk)))
        if n_chunks == 1:
            cuts = [0, None]                               # nothing to cut: the arrays go up as they are
        elif is_csr:
            cuts = [int(indptr64[b]) for b in bounds]
        else:
            cuts = [int(c) for c in np.searchsorted(user, np.asarray(bounds))]
            # the chunks are cut on the assumption that the triplets are sorted by user (the reference asserts it,
            # models.py:246): inside a chunk the ingest kernel verifies it, across the cuts it is verified here
            for bnd, cut in zip(bounds[1:-1], cuts[1:-1]):
                if (cut > 0 and user[cut - 1] >= bnd) or (cut < len(user) and user[cut] < bnd):
                    raise AssertionError("calculations assume testset is sorted by users!")

        def upload(c):                                     # chunk c -> the device, on the current stream
            a, b = bounds[c], bounds[c + 1]
            lo, hi = cuts[c], cuts[c + 1]
            head = (indptr64[a:b + 1].to(eng.device, non_blocking=True),) if is_csr else ()
            return head + tuple(t[lo:hi].to(eng.device, non_blocking=True) for t in host), a, b, lo

        def ingest(dev, a, b, lo):                         # -> the chunk's P and seen pattern
            if is_csr:
                ip, ix, vl = dev
                if lo:
                    eng.shift_i64(ip, -lo)                 # re-base the row pointers of the chunk
                p_dev = DeviceCSR(ip, ix if ix.dtype == torch.int32 else ix.to(torch.int32),
                                  vl if vl.dtype == torch.float32 else vl.to(torch.float32), (b - a, n_items))
                return p_dev, (p_dev.indptr, p_dev.indices)
            u_d, i_d, f_d = dev
            if a:
                eng.shift_i64(u_d, -a)                     # users of the chunk count from 0
            return self._test_csr_device(None, (b - a, n_items), stream_arrays=(u_d, i_d, f_d, None), sorted_users=True)

        if n_chunks == 1 and prof is None:
            return [ids.cpu().numpy() for ids in self._rank_lists(*ingest(*upload(0)), v_fold, v_score, ranks)]

        # fresh pinned result buffer: torch's caching host allocator re-uses the block once the previous result is
        # garbage-collected, so steady-state calls pay neither cudaHostAlloc nor page faults, and results never alias
        out = torch.empty((len(ranks), m, self.topk), dtype=torch.int64, pin_memory=True)
        main = torch.cuda.current_stream(eng.device)
        side = self.__dict__.setdefault("_copy_stream", torch.cuda.Stream(device=eng.device))
        back = self.__dict__.setdefault("_result_stream", torch.cuda.Stream(device=eng.device))

        def upload_aside(c):
            with torch.cuda.stream(side):
                dev, a, b, lo = upload(c)
                ev = torch.cuda.Event(enable_timing=prof is not None)
                ev.record(side)
            return (dev, ev, a, b, lo)

        t_host0 = time.perf_counter()

        def mark(stream):
            ev_ = torch.cuda.Event(enable_timing=True)
            ev_.record(stream)
            return ev_

        side.wait_stream(main)
        if prof is not None:
            ev_start = mark(main)
        nxt = upload_aside(0)
        keep = []
        for c in range(n_chunks):
            dev, ev, a, b, lo = nxt
            if c + 1 < n_chunks:
                nxt = upload_aside(c + 1)
            main.wait_event(ev)
            if prof is not None:
                prof.append(["chunk%d" % c, ev, mark(main), None, None, time.perf_counter() - t_host0])
            for t in dev:
                t.record_stream(main)                      # allocated on the side stream, consumed on the main one
            p_dev, seen = ingest(dev, a, b, lo)
            ids = self._rank_lists(p_dev, seen, v_fold, v_score, ranks)
            if prof is not None:
                prof[-1][3] = mark(main)
            scored = torch.cuda.Event()
            scored.record(main)
            with torch.cuda.stream(back):                  # results leave on their own stream / copy engine
                back.wait_event(scored)
                for j, t in enumerate(ids):
                    out[j, a:b].copy_(t, non_blocking=True)
                done = torch.cuda.Event(enable_timing=prof is not None)
                done.record(back)
            if prof is not None:
                prof[-1][4] = done
            keep.append((p_dev, seen, ids))
        main.synchronize()
        back.synchronize()
        if prof is not None:
            # per chunk, ms after the start of the call: upload done, compute start, compute end, D2H done, host enqueue time
            self.last_score_timings = {
                "host_total_ms": (time.perf_counter() - t_host0) * 1e3, "setup_ms": (t_host0 - t_entry) * 1e3,
                "chunks": [[name, ev_start.elapsed_time(up), ev_start.elapsed_time(c0), ev_start.elapsed_time(c1),
                            ev_start.elapsed_time(d1), host_t * 1e3] for name, up, c0, c1, d1, host_t in prof]}
        return list(out.numpy())

    # ---- sampled evaluation (RandomSampleEvaluationSVDMixin, models.py:1095-1183) ---------------------------------------
    def sampled_recommendations(self, holdout_items, unseen_items=None, test_data=None, shape=None, n_unseen=None, seed=None,
                                holdout_users=None):
        """Rank every test user's holdout items against a sample of unseen items (the EIGENREC protocol): scores of the
        ``[n_users x holdout_size]`` holdout items and of the ``[n_users x n_unseen]`` sampled items come from one
        gather-dot over the resident factors (pb200_gather_dot = inner_product_at, lib/sparse.py:58-72), then the top-k
        POSITIONS in the concatenated ``[holdout | unseen]`` row are returned (``np.apply_along_axis(topsort, ...)``,
        models.py:1182): position < holdout_size means a holdout item was ranked there.

        ``unseen_items=None`` samples them on the fly as the reference does (models.py:1137-1156, 1169-1176): ``n_unseen``
        items per user, drawn by numba's sampler from the seeds ``SeedSequence(seed).generate_state(n_users)`` and
        excluding the user's test profile and holdout items, in the order of ``profile + holdout`` as scipy forms it (built
        on the host, an O(nnz) pass like the reference's; its time is left in ``last_sampled_timings``).  Draw, scoring
        and ranking are one kernel (the routine of pb200_sampled_topk, called through pb200_sampled_topk_ranks with the
        one live rank).  ``holdout_users`` (the holdout frame's user column) gives the
        holdout rows by user runs, as matrix_from_observations does (evaluation.py:45-61); default: ``holdout_size``
        consecutive entries per user."""
        if unseen_items is None and getattr(self, "shard", None) is not None:
            raise NotImplementedError("on-the-fly sampled evaluation on an item-sharded model")
        r_live = self.factors[self.data.fields.itemid].shape[1]
        return self._sampled_lists([r_live], holdout_items, unseen_items, test_data, shape, n_unseen, seed,
                                   holdout_users)[0]

    def sampled_rank_sweep(self, ranks, holdout_items, unseen_items=None, n_unseen=None, seed=None, holdout_users=None,
                           test_data=None, shape=None):
        """``sampled_recommendations`` at every rank of ``ranks`` on the current factors truncated to that rank (the loop
        of find_optimal_svd_rank, evaluation/pipelines.py:81-116, with the truncation of models.py:819-832), made once:
        one exclusion-list pass, one SpMM at the largest rank and, drawn on the fly, one kernel that draws each user's
        items once and ranks them at every rank (pb200_sampled_topk_ranks).  With pre-sampled ``unseen_items`` there is
        no draw to share: one gather-dot + top-k per rank on the leading columns of the same embeddings.  Arguments as
        ``sampled_recommendations``.  Returns ``{rank: positions}``.

        The embeddings are the leading columns of ``P V`` at the largest rank, as the reference takes them; in fp32 a
        column's sum order depends on the SpMM kernel its column group runs on, so the lists can differ from those of a
        model truncated to that rank in the last bits of near-tied scores (DESIGN.md section 4)."""
        ranks = self._sweep_ranks(ranks)
        lists = self._sampled_lists(ranks, holdout_items, unseen_items, test_data, shape, n_unseen, seed, holdout_users)
        return dict(zip(ranks, lists))

    def rank_sweep(self, ranks):
        """``get_recommendations`` (standard protocol) at every rank of ``ranks`` on the current factors truncated to that
        rank, made once: one test-data ingest, one SpMM at the largest rank (through the right item projector for a model
        that carries HybridSVD projectors), then the fused scoring kernel once per rank on the leading columns of the
        same embeddings, honouring ``filter_seen`` and ``score_kernel``.  Returns ``{rank: int64 [n_test_users x topk]}``.
        The test data are read as ``get_recommendations`` reads them (``_test_input``) and scored in one chunk.  Same
        note on the embeddings as ``sampled_rank_sweep``."""
        ranks = self._sweep_ranks(ranks)
        rows, shape, is_csr, _ = self._checked_test_input(self._test_input)
        with self.engine.score_kernel_scope(self.score_kernel):
            return dict(zip(ranks, self._chunked_lists(rows, shape, is_csr, [0, shape[0]], ranks)))

    def _sweep_ranks(self, ranks):
        """the distinct ranks of a sweep, ascending; each must be a truncation of the current factors."""
        if getattr(self, "shard", None) is not None:
            raise NotImplementedError("rank sweep on an item-sharded model")
        ranks = sorted({int(r) for r in ranks})
        width = self.factors[self.data.fields.itemid].shape[1]
        if not ranks or ranks[0] < 1 or ranks[-1] > width:
            raise ValueError("sweep ranks must be in 1..%d, the width of the current factors (a larger rank needs a "
                             "rebuild); got %s" % (width, ranks))
        return ranks

    def _sampled_lists(self, ranks, holdout_items, unseen_items, test_data, shape, n_unseen, seed, holdout_users):
        """the sampled protocol's top-k positions at each of the ascending ``ranks``, as a list."""
        eng = self.engine
        if test_data is None:
            test_data, shape, _ = self._get_test_data()
        f = self.data.fields
        p_dev, _ = self._test_csr_device(test_data, shape)
        v_dev = self._device_factor(f.itemid)
        e = eng.spmm(p_dev, v_dev, ell=ranks[-1])                    # user_factors = test_matrix.dot(item_factors), :1158
        if unseen_items is None:
            if n_unseen is None:
                raise ValueError("Number of items to sample is unspecified.")
            hold = np.asarray(holdout_items, dtype=np.int64)
            hold = hold.reshape(shape[0], -1)
            if self.topk > hold.shape[1] + int(n_unseen):
                raise ValueError("topk exceeds the number of sampled items")
            t0 = time.perf_counter()
            indptr, indices = sampled_exclusion_lists(test_data, shape, hold, holdout_users)
            seeds = np.random.SeedSequence(seed).generate_state(int(shape[0]))
            t1 = time.perf_counter()
            pos = eng.sampled_topk_ranks(e, v_dev, ranks, eng.upload(hold), eng.upload(indptr), eng.upload(indices), seeds,
                                         int(n_unseen), self.topk)
            out = list(pos.cpu().numpy())
            self.last_sampled_timings = {"exclusion_ms": (t1 - t0) * 1e3, "device_ms": (time.perf_counter() - t1) * 1e3}
            return out
        items = np.concatenate([np.asarray(holdout_items, dtype=np.int64).reshape(shape[0], -1),
                                np.asarray(unseen_items, dtype=np.int64).reshape(shape[0], -1)], axis=1)
        if self.topk > items.shape[1]:
            raise ValueError("topk exceeds the number of sampled items")
        users = np.broadcast_to(np.arange(shape[0], dtype=np.int64)[:, None], items.shape)
        u_dev, i_dev = eng.upload(np.ascontiguousarray(users)), eng.upload(items)
        return [eng.topk_dense(eng.gather_dot(e, v_dev, r, u_dev, i_dev), self.topk).cpu().numpy() for r in ranks]

    # ---- item cold start (ItemColdStartSVDModelMixin.slice_recommendations, coldstart/models.py:216-222) ---------------
    def coldstart_recommendations(self, cold_item_features, feature_embeddings, transform_helper):
        """Top-k USERS for cold items: ``scores = (F_cold W) (W^T W)^+ (U diag(sigma))^T`` followed by
        ``get_topk_elements`` over users, ``filter_seen = False`` (coldstart/models.py:13-18, 216-222) -- the fused kernel
        with the roles swapped: the cold items' factors are the left operand, ``U diag(sigma)`` the right one.
        ``cold_item_features``: scipy sparse / dense [n_cold x n_features]; ``feature_embeddings`` W [n_features x r];
        ``transform_helper`` (W^T W)^+ [r x r] (``_item_features_transform_helper``).  Needs the user factors
        (``build(return_factors=True)``)."""
        import scipy.sparse as sps_
        eng = self.engine
        f = self.data.fields
        u = self.factors.get(f.userid, None)
        if u is None:
            raise ValueError("cold start needs the user factors: build(return_factors=True)")
        r = u.shape[1]
        w = np.asarray(feature_embeddings)[:, :r] @ np.asarray(transform_helper)[:r, :r]      # fold the r x r map into W
        fc = sps_.csr_matrix(cold_item_features)
        fc.sort_indices()
        ld = round_up(r, 32)
        w_pad = np.zeros((w.shape[0], ld), dtype=np.float32); w_pad[:, :r] = w
        if self.topk > u.shape[0]:
            raise ValueError("topk exceeds the number of users")
        us_dev = self._device_scaled_users()
        f_dev = eng.upload_csr(fc.indptr.astype(np.int64), fc.indices.astype(np.int32), fc.data.astype(np.float32), fc.shape)
        with eng.score_kernel_scope(self.score_kernel):
            e = eng.spmm(f_dev, eng.upload(w_pad), ell=ld)                  # cold item factors [n_cold x r]
            return eng.score_topk(e, us_dev, r, self.topk, seen=None).cpu().numpy()

    def _device_scaled_users(self):
        """``U diag(sigma)`` on the device, zero padded to a multiple of 32 columns, at the width of the arrays it was
        formed from; cached like ``_device_factor``.  Rank truncation (models.py:819-832) replaces U and sigma by their
        leading columns, views of the same arrays, so the cached operand serves every lower rank without an upload: its
        leading r columns are the truncated product's bits, and the scoring kernel reads r columns only."""
        f = self.data.fields
        u = np.asarray(self.factors[f.userid])
        s = np.asarray(self.factors["singular_values"])
        hit = self.__dict__.get("_dev_scaled_users")
        if hit is not None and _leading_columns_of(u, hit[0]) and _leading_columns_of(s, hit[1]):
            return hit[2]
        r = u.shape[1]
        us = np.zeros((u.shape[0], round_up(r, 32)), dtype=np.float32)
        us[:, :r] = u * s[None, :r]
        dev = self.engine.upload(us)
        self._dev_scaled_users = (u, s, dev)
        return dev

    def slice_recommendations(self, test_data, shape, start, stop, test_users=None):
        """Dense score rows for a (small) user slice -- kept for the single-user helpers
        (models.py:277-293,324-356).  Returns ``(scores float64 [m x n_items], slice_data)``."""
        user, item, fdbk = test_data
        sel = (user >= start) & (user < stop)
        sl = (user[sel] - start, item[sel], fdbk[sel])
        eng = self.engine
        p_dev, _ = self._test_csr_device(sl, (stop - start, shape[1]))
        v_dev = self._device_factor(self.data.fields.itemid)
        r_live = self.factors[self.data.fields.itemid].shape[1]
        e = eng.spmm(p_dev, v_dev, ell=r_live)
        s = eng.score_dense(e, v_dev, r_live)
        return s.cpu().numpy().astype(np.float64), sl


def _leading_columns_of(view, full):
    """True when ``view`` is ``full`` or ``full[..., :r]`` (what rank truncation makes of a factor, models.py:819-832):
    same memory start, same strides and leading dimensions, no wider."""
    if view is full:
        return True
    # numpy points a view at the array that owns the memory, or at ``full`` when ``full`` wraps a foreign buffer
    # (``Tensor.numpy()``)
    same_owner = view.base is full or (full.base is not None and view.base is full.base)
    return (same_owner and view.shape[:-1] == full.shape[:-1] and view.shape[-1] <= full.shape[-1]
            and view.strides == full.strides
            and view.__array_interface__["data"][0] == full.__array_interface__["data"][0])


def sampled_exclusion_lists(test_data, shape, holdout_items, holdout_users=None):
    """Per-user lists of the items the on-the-fly sampler excludes, in the ORDER the reference reads them:
    ``test_matrix + holdout_matrix`` (models.py:1145-1148) where test_matrix is get_test_matrix's CSR (zero feedback
    dropped, duplicates summed; models.py:196-211) and holdout_matrix the boolean CSR of matrix_from_observations
    (evaluation.py:45-61: indices in holdout order, rows = the runs of the holdout users).  scipy adds the two through its
    general path when a holdout row is unsorted, and the result's order is scipy's -- so scipy forms the sum here too.
    Returns ``(indptr int64, indices int32)``."""
    import scipy.sparse as sps_
    user, item, fdbk = test_data
    fdbk = np.asarray(fdbk)
    keep = fdbk != 0
    n_users, n_items = int(shape[0]), int(shape[1])
    profile = sps_.csr_matrix((fdbk[keep], (np.asarray(user)[keep], np.asarray(item)[keep])), shape=(n_users, n_items),
                              dtype=fdbk.dtype)
    hold = np.asarray(holdout_items).reshape(-1)
    if holdout_users is None:
        h = np.asarray(holdout_items).reshape(n_users, -1).shape[1]
        runs = np.arange(0, len(hold) + 1, max(h, 1), dtype=np.int64) if h else np.zeros(n_users + 1, np.int64)
    else:
        keys = np.asarray(holdout_users)
        runs = np.r_[0, np.where(np.diff(keys))[0] + 1, len(keys)].astype(np.int64)
    hm = sps_.csr_matrix((n_users, n_items), dtype=bool)
    hm.data, hm.indices, hm.indptr = np.ones(len(hold), dtype=bool), hold, runs
    s = profile + hm
    return s.indptr.astype(np.int64), s.indices.astype(np.int32)


def sampled_protocol_inputs(model):
    """What the sampled protocol reads from a ``RandomSampleEvaluationMixin`` data model (data.py:938-993,
    models.py:1095-1183): ``(holdout_items [n_users x holdout_size], unseen_items, kwargs)`` -- ``unseen_items`` the
    pre-sampled items of ``set_unseen_interactions`` with empty ``kwargs``, or None with the on-the-fly draw's
    ``n_unseen`` / ``seed`` / ``holdout_users``."""
    data = model.data
    userid, itemid = data.fields.userid, data.fields.itemid
    holdout = data.test.holdout
    assert data.holdout_size >= 1                               # models.py:1106
    holdout_items = holdout[itemid].values.reshape(-1, data.holdout_size)
    if data.unseen_interactions is None:
        if data.unseen_items_num is None:
            raise ValueError('Number of items to sample is unspecified.')     # models.py:1171-1172
        return holdout_items, None, dict(n_unseen=data.unseen_items_num, seed=data.seed,
                                         holdout_users=holdout[userid].values)
    test_users = holdout[userid].drop_duplicates().values      # preserve sorted (models.py:1123)
    unseen = np.concatenate(data.unseen_interactions.loc[test_users].values).reshape(len(test_users), data.unseen_items_num)
    return holdout_items, unseen, {}


def round_tucker_core(core, mode, rank):
    """Rank reduction of one mode of a Tucker core (CoffeeModel.round_core, models.py:966-980): thin SVD of the mode
    unfolding, keep the leading ``rank`` directions.  Returns ``(rotation [r_mode x rank], new_core)``.  Host numpy on
    purpose: the core is a few thousand numbers (<= 60 x 60 x 5) and the reference does this on the host as well."""
    moved = np.moveaxis(np.asarray(core), mode, 0)                  # [r_mode, remaining modes in their order]
    flat = moved.reshape((moved.shape[0], -1), order="F")
    u, s, vt = np.linalg.svd(flat, full_matrices=False)
    small = (s[:rank, None] * vt[:rank]).reshape((rank,) + moved.shape[1:], order="F")
    return u[:, :rank], np.moveaxis(small, 0, mode)


def csr_row_block(indptr, indices, values, shape, lo, hi):
    """rows [lo, hi) of a host CSR (numpy arrays or torch tensors) as a CSR of its own (views, re-based pointers)."""
    a, b = int(indptr[lo]), int(indptr[hi])
    return indptr[lo:hi + 1] - a, indices[a:b], values[a:b], (hi - lo, shape[1])


def stream_schedule(m, unit, first=0.06, growth=1.6):
    """Chunk bounds for the streamed path.  Chunks are whole waves of the scoring grid (``unit`` users = one 128-user
    tile per SM); the first is small so that little of the upload is exposed, each next one grows by at most ``growth``
    (< compute time / upload time per user, so the copy of chunk i+1 always hides behind the scoring of chunk i)."""
    waves = m / float(unit)
    if waves <= 2.0:
        return [0, m]
    size = max(1.0, round(waves * first))
    bounds, done = [0], 0.0
    while True:
        rest = waves - done
        if rest <= size * (1.0 + growth):              # the remainder fits one last chunk without starving the pipeline
            bounds.append(m)
            return bounds
        done += size
        bounds.append(int(done) * unit)
        size = float(int(size * growth + 0.999))


class _SVDState:
    """rank handling of SVDModel (models.py:802-832)."""

    def _init_svd_state(self):
        self._rank = host.DEFAULTS["svd_rank"]
        self.method = "PureSVD"
        self.factors = {}

    @property
    def rank(self):
        return self._rank

    @rank.setter
    def rank(self, new_value):
        if new_value != self._rank:
            self._rank = new_value
            self._check_reduced_rank(new_value)
            self._recommendations = None

    def _check_reduced_rank(self, rank):
        for entity, factor in self.factors.items():
            if factor is None:
                continue
            if factor.shape[-1] < rank:
                self._is_ready = False
                self.factors = dict.fromkeys(self.factors.keys())
                break
            else:
                self.factors = dict(**self.factors)
                self.factors[entity] = factor[..., :rank]


class B200SVDModel(_SVDDeviceMixin, _SVDState, host.RecommenderModel):
    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self._init_svd_state()

    def build(self, operator=None, return_factors="vh"):
        return _SVDDeviceMixin.build(self, operator=operator, return_factors=return_factors)


class _ScaledMatrixMixin:
    """ScaledMatrixMixin (models.py:864-895): column / row scaling of the training matrix, applied on the device by
    ``_SVDDeviceMixin._scaled``."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self._col_scaling = 0.4
        self._row_scaling = 1
        self.method = f"{self.method}-s"

    @property
    def col_scaling(self):
        return self._col_scaling

    @col_scaling.setter
    def col_scaling(self, new_value):
        if new_value != self._col_scaling:
            self._col_scaling = new_value
            self._recommendations = None

    @property
    def row_scaling(self):
        return self._row_scaling

    @row_scaling.setter
    def row_scaling(self, new_value):
        if new_value != self._row_scaling:
            self._row_scaling = new_value
            self._recommendations = None


class B200ScaledSVD(_ScaledMatrixMixin, B200SVDModel):
    """ScaledMatrixMixin + SVDModel (models.py:864-898)."""


# ------------------------------------------------------------------ HybridSVD ----------
def cholesky_factor_parts(factor):
    """``(L, perm)`` of a Cholesky factor ``K = P^T L`` of a similarity matrix, ``L L^T = P (S + beta I) P^T``: polara's
    ``CholeskyFactor`` (lib/cholesky.py; ``.L`` and the CHOLMOD factor's ``P()``) or an ``(L, perm)`` pair.  ``L`` comes
    back as a float64 CSR with sorted indices, ``perm`` as int64.  None stays None (that side is the identity)."""
    if factor is None:
        return None
    import scipy.sparse as sps_
    if isinstance(factor, (tuple, list)):
        lower, perm = factor
    else:
        lower, perm = factor.L, factor._factor.P()
    lower = sps_.csr_matrix(lower, dtype=np.float64)
    lower.sum_duplicates()
    lower.sort_indices()
    perm = np.asarray(perm, dtype=np.int64).ravel()
    n = lower.shape[0]
    if lower.shape[1] != n or perm.shape[0] != n or not np.array_equal(np.sort(perm), np.arange(n)):
        raise ValueError("a Cholesky factor needs a square L and a permutation of its %d rows; got L %s and %d entries"
                         % (n, lower.shape, perm.shape[0]))
    return lower, perm


def cholesky_operator(lower, perm):
    """the CSR of ``K = P^T L`` (host, float64): ``K v = apply_Pt(L v)`` puts row i of ``L`` at row ``perm[i]``."""
    inv = np.empty_like(perm)
    inv[perm] = np.arange(perm.shape[0], dtype=perm.dtype)
    k = lower[inv]
    k.sort_indices()
    return k


def hybrid_item_projectors(lower, perm, v):
    """build_item_projector (hybrid/models.py:315-326) in float64 on the host: ``(left, right) = (K^-T v, K v)`` with
    ``K^-T v = apply_Pt(L^-T v)`` (``chol.T.solve``, a triangular solve with ``L^T``) and ``K v = apply_Pt(L v)``
    (``chol.dot``).  Runs once per build."""
    from scipy.sparse.linalg import spsolve_triangular
    v = np.asarray(v, dtype=np.float64)
    right = np.empty_like(v)
    right[perm] = lower @ v
    left = np.empty_like(v)
    left[perm] = spsolve_triangular(lower.T.tocsr(), v, lower=False)
    return left, right


def _rescale_host(matrix, scaling, axis):
    """rescale_matrix (preprocessing/matrices.py:71-93, binary=True) on a float64 CSR: the lines along ``axis`` scaled by
    ``sqrt(count) ** (scaling - 1)``, ``count`` the line's stored entries.  The reference's sparse product with
    ``diags(...)`` stores only nonzero results, even at ``scaling == 1``, so the result holds no explicit zeros: after
    the row pass the column counts exclude the stored zeros the row counts include (as pb200_rescale counts them)."""
    import scipy.sparse as sps_
    norm = np.sqrt(np.asarray(matrix.getnnz(axis=axis)).ravel().astype(np.float64))
    factor = np.ones_like(norm)
    factor[norm != 0] = np.power(norm[norm != 0], scaling - 1)
    d = sps_.diags(factor)
    out = (matrix @ d).tocsr() if axis == 0 else (d @ matrix).tocsr()
    out.eliminate_zeros()
    return out


class _HybridSVDDeviceMixin(_SVDDeviceMixin):
    """Device implementation of HybridSVD.build (hybrid/models.py:352-388): the truncated SVD of ``K_u^T A K_i`` for the
    Cholesky factors ``K = P^T L`` of the user and item similarity matrices (either may be None: identity).  Without
    ``precompute_auxiliary_matrix`` the operator is never formed: the subspace iteration applies the three factors in
    turn (pb200_rsvd_factored); with it the product is formed on the host by scipy and factorised as an explicit
    operator (``build(operator=...)``).  The item projectors of the scoring step are then computed on the host in
    float64, as the reference computes them."""

    def _host_training_matrix(self):
        """get_training_matrix(dtype=np.float64) (models.py:160-177, 891-895 for the scaled variant) as a float64 CSR."""
        getter = getattr(self, "get_training_matrix", None)
        if getter is not None:
            return getter(dtype=np.float64)
        import scipy.sparse as sps_
        idx, val, shape = self.data.to_coo(tensor_mode=False, feedback_threshold=self.feedback_threshold)
        idx = _as_index_array(idx)
        m = sps_.coo_matrix((np.asarray(val, dtype=np.float64), (idx[:, 0], idx[:, 1])), shape=shape).tocsr()
        if hasattr(self, "_col_scaling"):
            m = _rescale_host(_rescale_host(m, self.row_scaling, 1), self.col_scaling, 0)
        return m

    def _device_factor_pair(self, lower, perm):
        """``(K, K^T)`` on the device: K formed on the host from L and perm (float32 values), K^T by pb200_csr_transpose."""
        eng = self.engine
        k = cholesky_operator(lower, perm)
        k_dev = eng.upload_csr(k.indptr.astype(np.int64), k.indices.astype(np.int32), k.data.astype(np.float32), k.shape)
        return k_dev, eng.transpose(k_dev)

    def build(self, return_factors="vh"):
        if not getattr(self, "_sparse_mode", True):
            raise NotImplementedError("Check the installation of scikit-sparse package.")
        if self._build_rows(1) is not None:
            raise NotImplementedError("row-sharded build of HybridSVD")
        # the order matters, as in the reference: reading the training data may fire the data model's change events,
        # which reset the Cholesky factors
        if self.precompute_auxiliary_matrix:
            svd_matrix = self._host_training_matrix()
        else:
            a = self._training_csr_device()
        items = cholesky_factor_parts(self.item_cholesky_factor)
        users = cholesky_factor_parts(self.user_cholesky_factor)
        if self.precompute_auxiliary_matrix:
            if items is not None:
                svd_matrix = (svd_matrix @ cholesky_operator(*items)).tocsr()
            if users is not None:
                svd_matrix = (cholesky_operator(*users).T @ svd_matrix).tocsr()
            _SVDDeviceMixin.build(self, operator=svd_matrix, return_factors=return_factors)
        else:
            item_pair = None if items is None else self._device_factor_pair(*items)
            user_pair = None if users is None else self._device_factor_pair(*users)
            self._build_factors(self.engine, return_factors, False, a=a, item_factor=item_pair, user_factor=user_pair)
        self.build_item_projector(self.factors[self.data.fields.itemid])
        self._clear_cholesky_cache()

    def build_item_projector(self, v):
        items = cholesky_factor_parts(self.item_cholesky_factor)
        if items is not None:
            itemid = self.data.fields.itemid
            left, right = hybrid_item_projectors(items[0], items[1], v)
            self.factors["%s_projector_left" % itemid] = left
            self.factors["%s_projector_right" % itemid] = right


class B200HybridSVD(_HybridSVDDeviceMixin, _SVDState, host.RecommenderModel):
    """Stand-alone HybridSVD (hybrid/models.py:335-394).  ``item_cholesky_factor`` / ``user_cholesky_factor``: polara's
    ``CholeskyFactor`` or an ``(L, perm)`` pair with ``L L^T = P (S + beta I) P^T`` and ``P v = v[perm]``; None (the
    default) leaves that side of the operator the identity.  Computing the factorisation is the caller's."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self._init_svd_state()
        self.method = "HybridSVD"
        self.precompute_auxiliary_matrix = False
        self.item_cholesky_factor = None
        self.user_cholesky_factor = None

    def build(self, return_factors="vh"):
        return _HybridSVDDeviceMixin.build(self, return_factors=return_factors)

    def _clear_cholesky_cache(self):
        """hybrid/models.py:241-247: a CholeskyFactor drops its cached L (an ``(L, perm)`` pair is the caller's)."""
        for factor in (self.item_cholesky_factor, self.user_cholesky_factor):
            if factor is not None and hasattr(factor, "_L"):
                factor._L = None


class B200ScaledHybridSVD(_ScaledMatrixMixin, B200HybridSVD):
    """ScaledHybridSVD (hybrid/models.py:397): HybridSVD on the scaled training matrix."""


# ------------------------------------------------------------------ item cold start ----------
class _ItemColdStartMixin:
    """Item cold start on the SVD family: a restatement of polara/recommender/coldstart/models.py, whose module cannot be
    imported without ``lightfm`` (its line 8 imports LightFMWrapper).  It composes, in this order:

    * ItemColdStartEvaluationMixin (:13-18): nothing is seen, and the lists are matched as (cold item, user) pairs:
      ``_prediction_key = '<itemid>_cold'``, ``_prediction_target = userid``;
    * ItemColdStartRecommenderMixin (:21-52): one row per cold item of ``index.itemid.cold_start``, the top-k users;
    * ItemColdStartSVDModelMixin (:149-222): the build with the user factors, then the feature mapping
      ``W = F^T V`` (``<itemid>_features`` in ``factors``, so rank truncation cuts it with the rest) and its transform
      ``pinv(W^T W)``, both once per build on the host in float64.  Scores are ``(F_cold W) pinv(W^T W) (U diag s)^T``.

    The device work is the parent's build and ``coldstart_recommendations`` (pb200_spmm_csr for the cold items' factors,
    pb200_score_topk over the users).  ``_mapping_source`` names the factor W is built from: the item factors V
    (SVDModelItemColdStart, :233-236) or HybridSVD's right item projector (HybridSVDItemColdStart, :247-251).

    Features: a DataFrame of per-item label lists (the reference's form, one-hot encoded by polara's ``stack_features``),
    or, with :class:`polara_b200.host.ColdStartData`, the data model's F and F_cold."""

    _mapping_source = "{}"

    def __init__(self, *args, item_features=None, **kwargs):
        super().__init__(*args, **kwargs)
        self.filter_seen = False                      # there are no seen entities in cold start
        self._prediction_key = "{}_cold".format(self.data.fields.itemid)
        self._prediction_target = self.data.fields.userid
        if item_features is None:                     # features are provided via the data model
            item_features = self.data.item_features
        assert item_features is not None
        self.item_features = item_features
        self.item_features_labels = None
        self._item_features_transform_helper = None
        self.data.subscribe(self.data.on_change_event, self._clean_metadata)

    def _clean_metadata(self):
        self.item_features_labels = None

    @property
    def item_features_embeddings(self):
        return self.factors.get("{}_features".format(self.data.fields.itemid), None)

    def _round_item_features_transform(self):
        try:
            rank = self.item_features_embeddings.shape[1]
        except AttributeError:                        # embeddings are None (not built, or cleared by a higher rank)
            self._item_features_transform_helper = None
        else:
            if self._item_features_transform_helper.shape[0] > rank:
                self.update_item_features_transform()
            else:
                raise ValueError("Unable to round: the rank of factors is not lower than the rank of transform!")

    def _check_reduced_rank(self, rank):
        super()._check_reduced_rank(rank)
        self._round_item_features_transform()

    def _features_given_as_matrix(self):
        import scipy.sparse as sps_
        return sps_.issparse(self.item_features)

    def encode_item_features(self):
        """the training items' one-hot F (:185-190)."""
        if self._features_given_as_matrix():
            return self.item_features
        from polara.lib.similarity import stack_features
        training_items = self.data.index.itemid.training.old.values
        item_features = self.item_features.reindex(training_items, fill_value=[])
        item_one_hot, self.item_features_labels = stack_features(item_features, stacked_index=False, normalize=False)
        return item_one_hot

    def encode_cold_item_features(self):
        """F_cold in the order of ``index.itemid.cold_start``, features unseen in training dropped (:26-29, 210-214)."""
        if self._features_given_as_matrix():
            return self.data.cold_item_features
        from polara.lib.similarity import stack_features
        cold_item_meta = self.item_features.reindex(self.data.index.itemid.cold_start.old.values, fill_value=[])
        cold_item_features, _ = stack_features(cold_item_meta, labels=self.item_features_labels, normalize=False)
        return cold_item_features

    def compute_item_features_mapping(self, item_features):
        return item_features.T.dot(self.factors[self._mapping_source.format(self.data.fields.itemid)])

    def update_item_features_transform(self):
        mapping = self.item_features_embeddings
        self._item_features_transform_helper = np.linalg.pinv(mapping.T @ mapping)

    def prepare_item_features_transformation(self):
        item_one_hot = self.encode_item_features()
        self.factors["{}_features".format(self.data.fields.itemid)] = self.compute_item_features_mapping(item_one_hot)
        self.update_item_features_transform()

    def build(self, *args, **kwargs):
        super().build(*args, return_factors=True, **kwargs)
        self.prepare_item_features_transformation()

    def get_recommendations(self):
        if self.verify_integrity and hasattr(self, "verify_data_integrity"):
            self.verify_data_integrity()
        return self.coldstart_recommendations(self.encode_cold_item_features(), self.item_features_embeddings,
                                              self._item_features_transform_helper)


class _HybridColdStartSource:
    _mapping_source = "{}_projector_right"


class B200SVDModelItemColdStart(_ItemColdStartMixin, B200SVDModel):
    """SVDModelItemColdStart (coldstart/models.py:225-236) on :class:`polara_b200.host.ColdStartData`."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.method = "PureSVD(cs)"

    def build(self, *args, **kwargs):
        return _ItemColdStartMixin.build(self, *args, **kwargs)


class B200ScaledSVDItemColdStart(_ScaledMatrixMixin, B200SVDModelItemColdStart):
    """ScaledSVDItemColdStart (coldstart/models.py:254)."""


class B200HybridSVDItemColdStart(_HybridColdStartSource, _ItemColdStartMixin, B200HybridSVD):
    """HybridSVDItemColdStart (coldstart/models.py:239-251): W is built from the right item projector, so a model
    without an item Cholesky factor (no projectors) has nothing to map the features with and raises KeyError, as the
    reference does."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.method = "HybridSVD(cs)"

    def build(self, *args, **kwargs):
        return _ItemColdStartMixin.build(self, *args, **kwargs)


class B200ScaledHybridSVDItemColdStart(_ScaledMatrixMixin, B200HybridSVDItemColdStart):
    """ScaledHybridSVDItemColdStart (coldstart/models.py:257)."""


# ------------------------------------------------------------------ CoFFee ----------
def flatten_weights(w, flattener):
    """``flatten_scores(w.T, flattener)`` (models.py:983-1006,1052) for the flatteners that are
    linear in the scores; returns the vector ``wt_flat`` [r2]."""
    wt = np.asarray(w).T
    if flattener is None:
        flattener = slice(None)
    if isinstance(flattener, str):
        if flattener not in ("sum", "mean"):
            raise NotImplementedError("only linear flatteners run on the device path")
        return getattr(np, flattener)(wt, axis=-1)
    if isinstance(flattener, int):
        return wt[..., flattener]
    if isinstance(flattener, (list, slice)):
        return np.sum(wt[..., flattener], axis=-1)
    if isinstance(flattener, tuple):
        sl, how = flattener
        if how not in ("sum", "mean"):
            raise NotImplementedError("only linear flatteners run on the device path")
        return getattr(np, how)(wt[..., sl or slice(None)], axis=-1)
    raise NotImplementedError("callable flatteners need dense tensor scores; not available on the device path")


class _CoffeeDeviceMixin(_DeviceModelMixin):
    """Device implementation of CoffeeModel.build (-> hooi, polara/lib/tensor.py:37-96) and
    CoffeeModel scoring (models.py:1042-1054)."""

    def _hooi_device(self, idx, val, shape, mlrank, init=None):
        """HOOI (polara/lib/tensor.py:37-96) on the device.  With ``self.shard`` set (world > 1) the nnz are sharded by
        user (SURVEY.md 8e): the mode-0 unfolding and ``u0`` hold this rank's users only (its Gram matrix is summed over
        the ranks inside pb200_tall_svd), the mode-1 / mode-2 TTM outputs are all-reduced and factored redundantly."""
        eng = self.engine
        r0, r1, r2 = mlrank
        n0, n1, n2 = (int(s) for s in shape)
        shard = getattr(self, "shard", None)
        sharded = shard is not None and shard.world > 1
        n0_all = n0
        if sharded:
            import torch.distributed as dist
            lo, hi = shard.user_range(n0)
            keep = (idx[:, 0] >= lo) & (idx[:, 0] < hi)
            idx = idx[keep].copy()
            idx[:, 0] -= lo
            val = np.asarray(val)[keep]
            n0 = hi - lo
        i0 = eng.upload(idx[:, 0].astype(np.int32))
        i1 = eng.upload(idx[:, 1].astype(np.int32))
        i2 = eng.upload(idx[:, 2].astype(np.int32))
        vals = eng.upload(np.asarray(val, dtype=np.float32))
        g0 = eng.coo_group(i0, n0, i1, i2, vals)        # seg, i1, i2, val grouped by user
        g1 = eng.coo_group(i1, n1, i0, i2, vals)        # grouped by item
        g2 = eng.coo_group(i2, n2, i0, i1, vals)        # grouped by feedback level
        if init is None:
            # same start as the reference (lib/tensor.py:57-63): RandomState(seed).rand + QR, on the host
            rs = np.random if self.seed is None else np.random.RandomState(self.seed)
            u1 = np.linalg.qr(rs.rand(n1, r1), mode="reduced")[0]
            u2 = np.linalg.qr(rs.rand(n2, r2), mode="reduced")[0]
        else:
            u1, u2 = init
        u1_d = eng.upload(np.ascontiguousarray(u1, dtype=np.float32))
        u2_d = eng.upload(np.ascontiguousarray(u2, dtype=np.float32))
        norm_old = 0.0
        trace = []
        for it in range(self.num_iters):
            # mode 0: res[i0, a(u2), b(u1)]  (ttm(..., u2, u1, ((2,0),(1,0))), tensor.py:70)
            unf = eng.ttm(n0, g0[0], g0[2], g0[1], g0[3], u2_d, r2, u1_d, r1)
            if sharded:
                eng.set_reduce_hook(dist.all_reduce)                 # rows of the unfolding are sharded: global Gram matrix
            try:
                u0_d, _, _ = self._tall_svd(unf, r2 * r1, r0)
            finally:
                if sharded:
                    eng.set_reduce_hook(None)
            # mode 1: res[i1, a(u2), b(u0)]  (tensor.py:74)
            unf = eng.ttm(n1, g1[0], g1[2], g1[1], g1[3], u2_d, r2, u0_d, r0)
            if sharded:
                dist.all_reduce(unf)                                  # every rank holds part of every item's nnz
            u1_d, _, _ = self._tall_svd(unf, r2 * r0, r1)
            # mode 2: res[i2, a(u1), b(u0)] (tensor.py:78) -- few huge segments; work on the transpose
            small = eng.ttm_reduce(n2, g2[0], g2[2], g2[1], g2[3], u1_d, r1, u0_d, r0)     # [n2 x r1*r0]
            if sharded:
                dist.all_reduce(small)
            small_t = small.t().contiguous()                                                 # [r1*r0 x n2]
            vv_d, ss, uut = self._tall_svd(small_t, n2, r2, want_vt=True)                    # left vecs of M^T = vv
            u2_d = uut.t().contiguous()                                                      # [n2 x r2]
            ss_h = ss.cpu().numpy()
            norm_new = float(np.linalg.norm(ss_h))
            trace.append(norm_new)
            growth = (norm_new - norm_old) / norm_new
            norm_old = norm_new
            if growth < self.growth_tol:
                break
        # core (tensor.py:90-92): rows of (ss * vv^T) are already descending here
        vv = vv_d[:, :r2].cpu().numpy().astype(np.float64)            # [r1*r0 x r2]
        core = (ss_h[:, None] * vv.T).reshape(r2, r1, r0).transpose(2, 1, 0)
        to_host = lambda t, r: t[:, :r].cpu().numpy().astype(np.float64)   # noqa: E731
        if sharded:
            full = torch.zeros((n0_all, u0_d.shape[1]), dtype=u0_d.dtype, device=u0_d.device)
            full[lo:hi].copy_(u0_d)
            dist.all_reduce(full)                                     # assemble the user factors (disjoint row blocks)
            u0_d = full
        return to_host(u0_d, r0), to_host(u1_d, r1), to_host(u2_d, r2), np.ascontiguousarray(core), trace

    def _tall_svd(self, m, width, rank, want_vt=False):
        eng = self.engine
        u, s, vt = eng.tall_svd(m if m.shape[1] == width else m[:, :width], rank, want_vt=want_vt)
        return u, s, vt

    def build(self):
        idx, val, shp = self.data.to_coo(tensor_mode=True)
        t0 = time.perf_counter()
        u0, u1, u2, core, trace = self._hooi_device(idx, val, shp, self.mlrank)
        self.engine.sync()
        t1 = time.perf_counter()
        if self.training_time is not None:
            self.training_time.append(t1 - t0)
        if self.verbose:
            print("{} training time: {:.3f}s".format(self.method, t1 - t0))
        f = self.data.fields
        self.factors[f.userid] = u0
        self.factors[f.itemid] = u1
        self.factors[f.feedback] = u2
        self.factors["core"] = core
        self.core_norm_trace = trace

    def get_recommendations(self):
        (user, item, fdbk_idx), shape, _ = self._checked_test_input(self._get_test_data)
        f = self.data.fields
        w = self.factors[f.feedback]
        # E[u,:] = sum_{(i,f) in u} (w[f,:] . wt_flat) v[i,:]   (SURVEY.md §8a row A9)
        c = np.asarray(w) @ flatten_weights(w, self.flattener)
        weights = c[np.asarray(fdbk_idx, dtype=np.int64)].astype(np.float32)
        p_dev, seen_dev = self._test_csr_device((user, item, None), shape, values=weights)
        with self.engine.score_kernel_scope(self.score_kernel):
            ids = self._score(p_dev, seen_dev, self._device_factor(f.itemid), self.factors[f.itemid].shape[1])
        return ids.cpu().numpy()

    def tucker_rank_sweep(self, mlranks):
        """``get_recommendations`` at every multilinear rank ``(r1, r2, r3)`` of ``mlranks`` on the current factors
        rounded to that rank (``mlrank = t``, models.py:949-980), made from one test-data ingest.  Returns
        ``{(r1, r2, r3): int64 [n_test_users x topk]}``, honouring ``filter_seen``, ``flattener`` and ``score_kernel``.

        Per triple the core is rounded mode by mode on the host as ``_check_reduced_rank`` rounds it; the user factor,
        which scoring never reads, is not rotated.  The item factor is rotated on the device (pb200_rotate_factor, once
        per ``(r1, r2)``) only when ``r2`` is below its width; the feedback factor and the per-level weight table are
        formed on the host with the expressions of ``get_recommendations``, and the test matrix's values are rewritten
        from that table (pb200_csr_values_from_table).  At full item rank the lists are bit-identical to the per-triple
        path; below it the rotated factor is the fixed fp64 chain of pb200_rotate_factor where the per-triple path uses
        numpy's BLAS, so lists can differ at near-ties (DESIGN.md section 4).  With ``profile_phases`` set the phases of
        every triple are timed into ``last_sweep_timings``."""
        if getattr(self, "shard", None) is not None:
            raise NotImplementedError("Tucker-rank sweep on an item-sharded model")
        f = self.data.fields
        entities = (f.userid, f.itemid, f.feedback)
        w_full = self.factors[f.feedback]
        flatten_weights(w_full, self.flattener)                 # a flattener the device path lacks raises before any work
        triples = list(dict.fromkeys(tuple(int(r) for r in t) for t in mlranks))
        widths = [None if self.factors.get(e) is None else self.factors[e].shape[1] for e in entities]
        for t in triples:
            if len(t) != 3 or min(t) < 1 or any(w is not None and r > w for r, w in zip(t, widths)):
                raise ValueError("sweep ranks must be triples within %s, the widths of the current factors (a larger "
                                 "rank needs a rebuild); got %s" % (tuple(widths), t))
        (user, item, fdbk_idx), shape, _ = self._checked_test_input(self._get_test_data)
        eng = self.engine
        prof = getattr(self, "profile_phases", False)
        u_d, i_d = eng.upload(_as_index_array(user)), eng.upload(_as_index_array(item))
        levels = eng.upload(np.asarray(fdbk_idx, dtype=np.int64))
        p_dev, perm, run_ptr = eng.coo_to_csr_runs(u_d, i_d, None, shape[:2])
        seen_dev = (p_dev.indptr, p_dev.indices)              # values never drop entries here: one pattern for all
        v64, rotated, out, timings = None, {}, {}, []
        with eng.score_kernel_scope(self.score_kernel):
            for t in triples:
                clock = _PhaseClock(prof)
                core, rot = self.factors["core"], [None, None, None]
                for mode in range(3):
                    if widths[mode] is not None and widths[mode] > t[mode]:
                        rot[mode], core = round_tucker_core(core, mode, t[mode])
                w = w_full if rot[2] is None else w_full.dot(rot[2])
                table = (np.asarray(w) @ flatten_weights(w, self.flattener)).astype(np.float32)
                clock.mark("round_ms", host=True)
                v_dev = rotated.get(t[:2])
                if v_dev is None:
                    if rot[1] is None:
                        v_dev = self._device_factor(f.itemid)
                    else:
                        if v64 is None:
                            v64 = eng.upload(np.asarray(self.factors[f.itemid], dtype=np.float64))
                        v_dev = eng.rotate_factor(v64, eng.upload(rot[1]))
                    rotated[t[:2]] = v_dev
                clock.mark("rotate_ms")
                eng.csr_values_from_table(p_dev, perm, run_ptr, levels, eng.upload(table))
                clock.mark("rewrite_ms")
                e = eng.spmm(p_dev, v_dev, ell=round_up(t[1], 32))
                clock.mark("spmm_ms")
                ids = eng.score_topk(e, v_dev, t[1], self.topk, seen=seen_dev if self.filter_seen else None)
                clock.mark("score_ms")
                out[t] = ids.cpu().numpy()
                timings.append(clock.result(t))
        if prof:
            self.last_sweep_timings = timings
        return out


class _PhaseClock:
    """CUDA events (host clock for ``host=True``) between the phases of one sweep step; inert unless ``on``."""

    def __init__(self, on):
        self.on, self.marks = on, []
        if on:
            self.t_host = time.perf_counter()
            self.last = torch.cuda.Event(enable_timing=True)
            self.last.record()

    def mark(self, name, host=False):
        if not self.on:
            return
        ev = torch.cuda.Event(enable_timing=True)
        ev.record()
        if host:
            now = time.perf_counter()
            self.marks.append((name, (now - self.t_host) * 1e3))
        else:
            self.marks.append((name, (self.last, ev)))
        self.last = ev

    def result(self, key):
        if not self.on:
            return None
        torch.cuda.synchronize()
        return dict(mlrank=key, **{n: (v if isinstance(v, float) else v[0].elapsed_time(v[1])) for n, v in self.marks})


class B200CoffeeModel(_CoffeeDeviceMixin, host.RecommenderModel):
    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self._mlrank = host.DEFAULTS["mlrank"]
        self.factors = {}
        self.method = "CoFFee"
        self._flattener = host.DEFAULTS["flattener"]
        self.growth_tol = host.DEFAULTS["growth_tol"]
        self.num_iters = host.DEFAULTS["num_iters"]
        self.show_output = False
        self.seed = None
        self.parallel_ttm = True

    @property
    def mlrank(self):
        return self._mlrank

    @mlrank.setter
    def mlrank(self, new_value):
        if new_value != self._mlrank:
            self._mlrank = new_value
            self._check_reduced_rank(new_value)
            self._recommendations = None

    def _check_reduced_rank(self, mlrank):
        """models.py:949-963: lowering a mode's rank rotates its factor and shrinks the core (no rebuild); raising it
        invalidates the model."""
        for mode, entity in enumerate(self.data.fields):
            factor = self.factors.get(entity, None)
            if factor is None:
                continue
            rank = mlrank[mode]
            if factor.shape[1] < rank:
                self._is_ready = False
                self.factors = {}
                break
            if factor.shape[1] > rank:
                self.factors = dict(self.factors)             # a backup of the old dict stays untouched
                rotation, self.factors["core"] = round_tucker_core(self.factors["core"], mode, rank)
                self.factors[entity] = factor.dot(rotation)

    round_core = staticmethod(round_tucker_core)

    @property
    def flattener(self):
        return self._flattener

    @flattener.setter
    def flattener(self, new_value):
        if new_value != self._flattener:
            self._flattener = new_value
            self._recommendations = None

    def build(self):
        return _CoffeeDeviceMixin.build(self)


# ------------------------------------------------------------------ item-to-item ----------
def cooc_nnz_max(memory_hard_limit):
    """``get_nnz_max`` (lib/sparse.py:21-22): beyond this many stored scores a chunk's sparse block is made dense."""
    import sys
    per_entry = sys.getsizeof(()) + 2 * (sys.getsizeof(1.0) + np.dtype(np.intp).itemsize)
    return int(memory_hard_limit * (1024 ** 3) / per_entry)


def cooc_chunk_modes(nnz_u, n_items, topk, memory_hard_limit, dense_output=False):
    """The reference's user chunks for the item-to-item model and the form each chunk's score block takes there:
    ``[(start, stop, dense)]``.  Chunks: ``array_split`` (utils.py:7-53) with result width ``topk``, scores multiplier 1
    and float64 scores; ``get_available_memory()`` returns bytes that are read as GB, so the limit is exactly
    ``memory_hard_limit`` whenever it is set (and never binds otherwise).  Form (lib/sparse.py:25-55): dense with
    ``dense_output``, or when the chunk's nonzero scores ``sum(nnz_u)`` exceed ``cooc_nnz_max`` or half the block."""
    nnz_u = np.asarray(nnz_u, dtype=np.int64)
    m, n = int(nnz_u.shape[0]), int(n_items)
    chunk = m
    s0, s1 = m / 1024, n / 1024
    item_kb = np.dtype(np.float64).itemsize / 1024
    result_mem = s0 * (topk / 1024) * item_kb
    if memory_hard_limit and s0 * s1 * item_kb + result_mem > memory_hard_limit:
        chunk = min(int((memory_hard_limit - result_mem) / (s1 * item_kb * (1 / 1024) + item_kb / 1024 ** 2) - 1), chunk)
        if chunk <= 0:
            raise MemoryError()
    n_chunks = m // chunk + int(m % chunk > 0)
    size, rem = divmod(m, n_chunks)
    bounds = np.cumsum([0] + rem * [size + 1] + (n_chunks - rem) * [size])
    nnz_max = cooc_nnz_max(memory_hard_limit)
    out = []
    for a, b in zip(bounds[:-1].tolist(), bounds[1:].tolist()):
        nnz = int(nnz_u[a:b].sum())
        out.append((a, b, bool(dense_output or nnz > nnz_max or nnz > 0.5 * (b - a) * n)))
    return out


class _CooccurrenceDeviceMixin(_DeviceModelMixin):
    """Device implementation of CooccurrenceModel.build / get_recommendations (models.py:693-725, 391-405): S = A^T A
    stays on the device, as a dense fp64 matrix or as an fp64 CSR (``storage``); scoring computes every test user's
    ``P S`` row once and returns its list under the rule the reference's chunk of that user applies
    (``cooc_chunk_modes``).  Both forms give the same bits.

    ``storage``: ``"auto"`` builds S dense wherever it fits the device and sparse only where the dense build would
    refuse with MemoryError; ``"dense"`` always dense (and that refusal); ``"sparse"`` always the CSR."""

    storage = "auto"
    i2i_storage = None           # the form the last build took: "dense" | "sparse"

    def _memory_hard_limit(self):
        return host.DEFAULTS["memory_hard_limit"]

    def build(self):
        data = self.data
        idx, val, shape = data.to_coo(tensor_mode=False, feedback_threshold=self.feedback_threshold)
        if self.storage not in ("auto", "dense", "sparse"):
            raise ValueError("storage must be 'auto', 'dense' or 'sparse', got %r" % (self.storage,))
        eng = self.engine
        t0 = time.perf_counter()
        idx_d = eng.upload(np.ascontiguousarray(_as_index_array(idx)))
        a = eng.coo_to_csr(idx_d[:, 0], idx_d[:, 1], eng.upload(_as_value_array(val)), shape)
        self._i2i_dev = self._i2i_csr = None
        if self.storage != "sparse":
            try:
                self._i2i_dev = eng.cooc_build(a, implicit=self.implicit)
            except MemoryError:
                if self.storage == "dense":
                    raise
        if self._i2i_dev is None:
            self._i2i_csr = eng.cooc_build_csr(a, implicit=self.implicit)
        self.i2i_storage = "dense" if self._i2i_dev is not None else "sparse"
        self._i2i_items = int(shape[1])
        eng.sync()
        t1 = time.perf_counter()
        if self.training_time is not None:
            self.training_time.append(t1 - t0)          # track_time, models.py:703
        if self.verbose:
            print("{} training time: {:.3f}s".format(self.method, t1 - t0))

    def get_recommendations(self):
        test_data, shape, _ = self._checked_test_input(self._get_test_data)
        nnz, dense, sparse = self.i2i_lists(test_data, shape)
        out = np.empty((shape[0], self.topk), dtype=np.int64)
        for a, b, is_dense in cooc_chunk_modes(nnz, shape[1], self.topk, self._memory_hard_limit(), self.dense_output):
            out[a:b] = dense[a:b] if is_dense else sparse[a:b]
        return out

    def _scoring_csr(self):
        """the fp64 CSR the sparse form scores with (P S_csr), or None for the dense form"""
        return self._i2i_csr

    def _scoring_test_csr(self, test_data, shape):
        return self._test_csr_device(test_data, shape)

    def i2i_lists(self, test_data, shape):
        """``(nnz_u, dense-rule lists, sparse-rule lists)`` of the test users, as numpy arrays (pb200_i2i_topk or, for
        the sparse form, pb200_i2i_topk_csr)."""
        eng = self.engine
        p_dev, seen_dev = self._scoring_test_csr(test_data, shape)
        seen = seen_dev if self.filter_seen else None
        s_csr = self._scoring_csr()
        if s_csr is None:
            nnz, dense, sparse = eng.i2i_topk(self._i2i_dev, self._i2i_items, p_dev, self.topk, seen=seen,
                                              implicit=self.implicit)
        else:
            nnz, dense, sparse = eng.i2i_topk_csr(s_csr, p_dev, self.topk, seen=seen, implicit=self.implicit)
        return nnz.cpu().numpy(), dense.cpu().numpy(), sparse.cpu().numpy()


class B200CooccurrenceModel(_CooccurrenceDeviceMixin, host.RecommenderModel):
    """Stand-alone item-to-item model (CooccurrenceModel, models.py:693-725)."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.method = "item-to-item"
        self.implicit = False
        self.dense_output = False

    def build(self):
        return _CooccurrenceDeviceMixin.build(self)


def dropin_i2i():
    """``PolaraB200Cooccurrence``: the device item-to-item model on the REAL ``polara`` CooccurrenceModel; the chunk
    rules read ``polara.recommender.defaults.memory_hard_limit`` as the reference does."""
    from polara.recommender import defaults
    from polara.recommender.models import CooccurrenceModel

    class PolaraB200Cooccurrence(_CooccurrenceDeviceMixin, CooccurrenceModel):
        def _memory_hard_limit(self):
            return defaults.memory_hard_limit

        def build(self):
            return _CooccurrenceDeviceMixin.build(self)

    return PolaraB200Cooccurrence


class _SimilarityDeviceMixin(_CooccurrenceDeviceMixin):
    """Device implementation of SimilarityAggregation (hybrid/models.py:25-44): the item relations of the data model
    with a zero diagonal and no stored zeros, scored as ``sparse_dot(P, S)`` -- ``P S^T`` (lib/sparse.py:48), so the
    device holds S^T as an fp64 CSR -- under the chunk rules of the item-to-item model.  With ``dense_output`` the
    reference multiplies through ``csc_matvec`` (lib/sparse.py:40-43), which reads the stored arrays of S as CSC: that
    is ``P S`` for relations held as CSR and ``P S^T`` for any other format, and the device follows it.  ``implicit``
    scores with ones for every nonzero test feedback (hybrid/models.py:41-42)."""

    def build(self):
        rel = self.data.item_relations.copy()        # the copy keeps the data model's matrix intact (:33)
        rel.setdiag(0)
        rel.eliminate_zeros()
        self.item_similarity_matrix = rel
        self._i2i_dev = None
        self._i2i_items = int(rel.shape[1])
        self._sim_forms = {}
        self._sim_operand_is_s = getattr(rel, "format", None) == "csr"
        self.i2i_storage = "sparse"

    def _scoring_csr(self):
        """S^T, or S for ``dense_output`` on CSR relations, as a device fp64 CSR (uploaded once per form)."""
        import scipy.sparse as sps
        use_s = bool(self.dense_output) and self._sim_operand_is_s
        hit = self._sim_forms.get(use_s)
        if hit is None:
            rel = self.item_similarity_matrix
            mat = sps.csr_matrix(rel if use_s else rel.T, dtype=np.float64)
            mat.sum_duplicates()
            mat.sort_indices()
            eng = self.engine
            hit = DeviceCSR(eng.upload(mat.indptr.astype(np.int64)), eng.upload(mat.indices.astype(np.int32)),
                            eng.upload(mat.data.astype(np.float64)), mat.shape)
            self._sim_forms[use_s] = hit
        return hit

    def _scoring_test_csr(self, test_data, shape):
        if not self.implicit:
            return self._test_csr_device(test_data, shape)
        user, item, fdbk = test_data
        # ones for the nonzero feedback; zero feedback is still dropped (get_test_matrix, models.py:197-201)
        ones = (np.asarray(fdbk) != 0).astype(np.float64)
        return self._test_csr_device((user, item, ones), shape)

    def i2i_lists(self, test_data, shape):
        eng = self.engine
        p_dev, seen_dev = self._scoring_test_csr(test_data, shape)
        seen = seen_dev if self.filter_seen else None
        # with ``implicit`` the values are already 1 (or a count of duplicate triplets, whose sign is 1)
        nnz, dense, sparse = eng.i2i_topk_csr(self._scoring_csr(), p_dev, self.topk, seen=seen, implicit=self.implicit)
        return nnz.cpu().numpy(), dense.cpu().numpy(), sparse.cpu().numpy()


class B200SimilarityAggregation(_SimilarityDeviceMixin, host.RecommenderModel):
    """Stand-alone SimilarityAggregation (hybrid/models.py:25-44) on a data model that carries ``item_relations``
    (``host.ArrayData(..., item_relations=...)``)."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.method = "SIM"
        self.implicit = False
        self.dense_output = False
        self.item_similarity_matrix = False

    def build(self):
        return _SimilarityDeviceMixin.build(self)


def dropin_similarity():
    """``PolaraB200SimilarityAggregation``: the device scorer on the REAL ``polara`` SimilarityAggregation (data models
    with item relations, e.g. SimilarityDataModel); the chunk rules read ``polara.recommender.defaults.memory_hard_limit``
    as the reference does."""
    from polara.recommender import defaults
    from polara.recommender.hybrid.models import SimilarityAggregation

    class PolaraB200SimilarityAggregation(_SimilarityDeviceMixin, SimilarityAggregation):
        def _memory_hard_limit(self):
            return defaults.memory_hard_limit

        def build(self):
            return _SimilarityDeviceMixin.build(self)

    return PolaraB200SimilarityAggregation


def dropin():
    """Returns ``(B200SVDModel, B200ScaledSVD, B200CoffeeModel)`` derived from the REAL
    ``polara`` classes (requires the reference package to be importable)."""
    from polara.recommender.models import CoffeeModel, ScaledSVD, SVDModel

    class PolaraB200SVD(_SVDDeviceMixin, SVDModel):
        def build(self, operator=None, return_factors="vh"):
            return _SVDDeviceMixin.build(self, operator=operator, return_factors=return_factors)

    class PolaraB200ScaledSVD(_SVDDeviceMixin, ScaledSVD):
        def build(self, operator=None, return_factors="vh"):
            return _SVDDeviceMixin.build(self, operator=operator, return_factors=return_factors)

    class PolaraB200Coffee(_CoffeeDeviceMixin, CoffeeModel):
        def build(self):
            return _CoffeeDeviceMixin.build(self)

    return PolaraB200SVD, PolaraB200ScaledSVD, PolaraB200Coffee


def dropin_hybrid():
    """``(PolaraB200HybridSVD, PolaraB200ScaledHybridSVD)``: the device HybridSVD build on the REAL ``polara`` HybridSVD
    and ScaledHybridSVD (hybrid/models.py:335-397).  The Cholesky factors come from polara's own CholeskyFactorsMixin
    (CHOLMOD on the host); the build follows HybridSVD.build, with the matrix-free operator on the device
    (pb200_rsvd_factored)."""
    from polara.recommender.hybrid.models import HybridSVD, ScaledHybridSVD

    class PolaraB200HybridSVD(_HybridSVDDeviceMixin, HybridSVD):
        def build(self, return_factors="vh"):
            return _HybridSVDDeviceMixin.build(self, return_factors=return_factors)

    class PolaraB200ScaledHybridSVD(_HybridSVDDeviceMixin, ScaledHybridSVD):
        def build(self, return_factors="vh"):
            return _HybridSVDDeviceMixin.build(self, return_factors=return_factors)

    return PolaraB200HybridSVD, PolaraB200ScaledHybridSVD


def dropin_coldstart():
    """``(PolaraB200SVDModelItemColdStart, PolaraB200ScaledSVDItemColdStart, PolaraB200HybridSVDItemColdStart,
    PolaraB200ScaledHybridSVDItemColdStart)``: the item cold-start models on the REAL ``polara`` SVDModel, ScaledSVD,
    HybridSVD and ScaledHybridSVD, for polara's ``ItemColdStartData`` (with item relations for the HybridSVD pair, e.g.
    ``ItemColdStartSimilarityData``).  ``polara.recommender.coldstart.models`` is not imported, so ``lightfm`` need not be
    installed; the features are one-hot encoded by polara's own ``stack_features``."""
    from polara.recommender.hybrid.models import HybridSVD
    from polara.recommender.models import ScaledMatrixMixin, SVDModel

    class PolaraB200SVDModelItemColdStart(_ItemColdStartMixin, _SVDDeviceMixin, SVDModel):
        def __init__(self, *args, **kwargs):
            super().__init__(*args, **kwargs)
            self.method = "PureSVD(cs)"

        def build(self, *args, **kwargs):
            return _ItemColdStartMixin.build(self, *args, **kwargs)

    class PolaraB200ScaledSVDItemColdStart(ScaledMatrixMixin, PolaraB200SVDModelItemColdStart):
        pass

    class PolaraB200HybridSVDItemColdStart(_HybridColdStartSource, _ItemColdStartMixin, _HybridSVDDeviceMixin,
                                           HybridSVD):
        def __init__(self, *args, **kwargs):
            super().__init__(*args, **kwargs)
            self.method = "HybridSVD(cs)"

        def build(self, *args, **kwargs):
            return _ItemColdStartMixin.build(self, *args, **kwargs)

    class PolaraB200ScaledHybridSVDItemColdStart(ScaledMatrixMixin, PolaraB200HybridSVDItemColdStart):
        pass

    return (PolaraB200SVDModelItemColdStart, PolaraB200ScaledSVDItemColdStart, PolaraB200HybridSVDItemColdStart,
            PolaraB200ScaledHybridSVDItemColdStart)


def dropin_sampled():
    """``PolaraB200SampledSVD``: the device path under the reference's ``RandomSampleEvaluationSVDMixin`` (models.py:1095-
    1183) for data models built with ``RandomSampleEvaluationMixin`` (data.py:938-993) whose unseen interactions were set
    with ``set_unseen_interactions``, or sampled on the fly (``unseen_interactions is None``, ``unseen_items_num`` set):
    the device draws the same items as numba's sampler (lib/sampler.py) from ``SeedSequence(data.seed)``, models.py:
    1169-1176.  An item-sharded model raises NotImplementedError there."""
    import pandas as pd
    from polara.recommender.models import RandomSampleEvaluationSVDMixin, SVDModel

    class PolaraB200SampledSVD(_SVDDeviceMixin, RandomSampleEvaluationSVDMixin, SVDModel):
        def build(self, operator=None, return_factors="vh"):
            return _SVDDeviceMixin.build(self, operator=operator, return_factors=return_factors)

        def get_recommendations(self):
            if self._prediction_target == self.data.fields.itemid:
                return _SVDDeviceMixin.get_recommendations(self)
            holdout_items, unseen, kwargs = sampled_protocol_inputs(self)
            return self.sampled_recommendations(holdout_items, unseen, **kwargs)

        def rank_sweep(self, ranks):
            """the lists of ``get_recommendations`` at every rank of ``ranks`` (``{rank: lists}``), dispatched on
            ``_prediction_target`` as ``get_recommendations`` is: the standard sweep for items, else the sampled one."""
            if self._prediction_target == self.data.fields.itemid:
                return _SVDDeviceMixin.rank_sweep(self, ranks)
            holdout_items, unseen, kwargs = sampled_protocol_inputs(self)
            return self.sampled_rank_sweep(ranks, holdout_items, unseen, **kwargs)

    return PolaraB200SampledSVD
