"""Host-side mirror of the reference's model/data protocol for the hot path.

The reference toolchain is Python, so the host side is Python too.  When the real
``polara`` package is importable the drop-in classes in :mod:`polara_b200.models`
subclass *its* ``SVDModel``/``CoffeeModel`` (see ``polara_b200.models.dropin``); on a
machine without it the classes below provide the same surface
(``build()``, ``get_recommendations()``, ``get_topk_elements()``, ``evaluate()``,
``recommendations``, ``rank``/``topk``/``filter_seen`` ...) with the same argument
meaning and error behaviour, citing the reference lines they mirror.
"""
from __future__ import annotations

from collections import namedtuple

import numpy as np

Fields = namedtuple("Fields", "userid itemid feedback")
_Index = namedtuple("Index", "userid itemid feedback")
_Test = namedtuple("TestData", "testset holdout")

# polara/recommender/defaults.py:5-51 (only what the hot path reads)
DEFAULTS = dict(topk=10, filter_seen=True, feedback_threshold=None, switch_positive=None,
                verify_integrity=True, max_test_workers=None, svd_rank=10, mlrank=(13, 10, 2),
                growth_tol=0.0001, num_iters=25, flattener=slice(0, None), ndcg_alternative=True,
                memory_hard_limit=1)


class ArrayData:
    """Minimal stand-in for ``polara.recommender.data.RecommenderData`` that replays the
    arrays the data model hands to a model (data.py:794-884): training COO, user-sorted
    test triplets, test shape and the holdout frame.  All splitting/reindexing logic of
    the reference is out of scope (SURVEY.md §2 row 5)."""

    on_change_event = "on_change"
    on_update_event = "on_update"

    def __init__(self, train_idx, train_val, train_shape, test_user=None, test_item=None, test_fdbk=None,
                 test_shape=None, holdout=None, warm_start=True, fields=("userid", "itemid", "rating"),
                 n_feedback=None, holdout_size=3, item_relations=None):
        self.fields = Fields(*fields)
        # item x item side relations (SimilarityDataModel.item_relations, hybrid/data.py:25-28), in the item index of
        # the training data; read by B200SimilarityAggregation
        self.item_relations = item_relations
        self._train = (np.asarray(train_idx), np.asarray(train_val), tuple(int(s) for s in train_shape))
        self._test_coo = None if test_user is None else (np.asarray(test_user), np.asarray(test_item),
                                                         np.asarray(test_fdbk))
        self._test_shape = None if test_shape is None else tuple(int(s) for s in test_shape)
        self.warm_start = warm_start
        self.test_sample = None
        self.holdout_size = holdout_size
        self.test = _Test(None, holdout)
        n_items = self._train[2][1]
        self.index = _Index(None, np.empty((n_items, 2)),
                            None if n_feedback is None else np.empty((n_feedback, 2)))
        self._subscribers = []
        # optional fast paths for very large problems (pinned host CSR, see models._csr_from_data)
        self.train_csr = None
        self.test_csr = None

    # events (data.py:35-76): nothing ever changes in a frozen replay
    def subscribe(self, event, callback):
        self._subscribers.append((event, callback))

    def to_coo(self, tensor_mode=False, feedback_threshold=None):
        idx, val, shp = self._train
        if tensor_mode != (idx.shape[1] == 3):
            raise ValueError("ArrayData holds %d-way training indices" % idx.shape[1])
        if feedback_threshold is not None:
            keep = val >= feedback_threshold          # data.py:783-788 (filter_values=True)
            idx, val = idx[keep], val[keep]
        return idx.astype(np.intp, copy=False), np.ascontiguousarray(val), shp

    def test_to_coo(self, tensor_mode=False, feedback_threshold=None):
        if self._test_coo is None:
            raise ValueError("Unable to read test data")       # data.py:840-841
        u, i, f = self._test_coo
        if feedback_threshold is not None and not tensor_mode:
            f = np.where(f >= feedback_threshold, f, 0)         # data.py:789-790 (filter_values=False)
        return u.astype(np.intp, copy=False), i.astype(np.intp, copy=False), f

    def get_test_shape(self, tensor_mode=False):
        shp = self._test_shape
        if shp is None:
            raise ValueError("Unable to read test data")
        if tensor_mode and len(shp) == 2:
            shp = shp + (self.index.feedback.shape[0],)
        return shp if tensor_mode else shp[:2]

    @classmethod
    def from_golden(cls, g):
        import pandas as pd
        hold = pd.DataFrame({"userid": g["holdout_user"], "itemid": g["holdout_item"], "rating": g["holdout_fdbk"]})
        tensor = g["train_idx"].shape[1] == 3
        return cls(g["train_idx"], g["train_val"], g["train_shape"], g["test_user"], g["test_item"],
                   g["test_fdbk"], g["test_shape"], holdout=hold,
                   warm_start=bool(g["warm_start"]) if "warm_start" in g else True,
                   n_feedback=int(g["train_shape"][2]) if tensor else None)


_ItemColdIndex = namedtuple("ItemIndex", "training cold_start")


class ColdStartData:
    """Stand-alone item cold-start data model: what ``ItemColdStartData`` (coldstart/data.py:10-224) hands to the SVD
    family's cold-start models once its split is made.  Splitting, reindexing and the one-hot encoding of DataFrame
    features are out of scope; the caller passes arrays in the model's index:

    * ``train_idx`` [nnz x 2] (user, item), ``train_val``, ``train_shape``: the training triplets of the warm items;
    * ``cold_item``, ``cold_user``, ``cold_fdbk``: the holdout, every interaction of the cold items, by cold id;
    * ``item_features`` F [n_items x n_features] and ``cold_item_features`` F_cold [n_cold x n_features] (row = cold
      id): one-hot features of the training and the cold items in one column space;
    * ``n_users``: the training users (the columns of the cold items' lists);
    * ``representative_users``: optional user ids (data.py:37-46).

    The rules of the reference's post-processing (data.py:128-217) are applied here:

    * the cold items are those with holdout rows;
    * a cold item none of whose features a training item has is dropped, with its holdout rows (data.py:162-185);
    * with ``representative_users``, when some cold item has no holdout row of a representative user, that item is
      dropped and the holdout keeps the representative users' rows only; when every cold item has one, the holdout
      stays whole (data.py:143-160, 187-210: the filter is only set up for items that lack one);
    * features no training item has are dropped from F_cold (``stack_features`` with the training labels drops
      unknown labels, similarity.py:259-267);
    * the holdout is sorted by cold id (data.py:212-217); ``index.itemid.cold_start`` holds the kept cold ids in
      ascending order, and ``cold_item_features`` their rows in that order.

    Scoring still ranks every training user for a cold item; the representative users only filter the holdout."""

    on_change_event = "on_change"
    on_update_event = "on_update"

    def __init__(self, train_idx, train_val, train_shape, cold_item, cold_user, cold_fdbk, item_features,
                 cold_item_features, n_users=None, representative_users=None, fields=("userid", "itemid", "rating")):
        import pandas as pd
        import scipy.sparse as sps
        self.fields = Fields(*fields)
        self._train = (np.asarray(train_idx), np.asarray(train_val), tuple(int(s) for s in train_shape))
        n_users = self._train[2][0] if n_users is None else int(n_users)
        f = sps.csr_matrix(item_features, dtype=np.float64)
        fc = sps.csr_matrix(cold_item_features, dtype=np.float64)
        if f.shape[0] != self._train[2][1] or fc.shape[1] != f.shape[1]:
            raise ValueError("item features must be [n_items x n_features] (%d items) and cold item features share their "
                             "columns; got %s and %s" % (self._train[2][1], f.shape, fc.shape))
        seen_cols = np.zeros(f.shape[1], dtype=bool)
        seen_cols[f.indices[f.data != 0]] = True
        fc = fc.multiply(seen_cols[None, :].astype(np.float64)).tocsr()      # unknown features dropped
        fc.eliminate_zeros()
        cold_item, cold_user = np.asarray(cold_item, dtype=np.int64), np.asarray(cold_user, dtype=np.int64)
        cold_fdbk = np.asarray(cold_fdbk)
        present = np.bincount(cold_item, minlength=fc.shape[0]) > 0          # the cold index comes from the holdout
        keep_item = present & (np.diff(fc.indptr) > 0)                       # shares a feature with a training item
        keep_row = keep_item[cold_item]
        if representative_users is not None:
            representative_users = np.unique(np.asarray(representative_users, dtype=np.int64))
            is_repr_row = np.isin(cold_user, representative_users)
            has_repr = np.zeros(fc.shape[0], dtype=bool)
            has_repr[cold_item[is_repr_row]] = True
            if not has_repr[present].all():          # data.py:158-159, 198-201: only then is the holdout filtered
                keep_item &= has_repr
                keep_row &= is_repr_row & keep_item[cold_item]
        order = np.argsort(cold_item[keep_row], kind="stable")
        cold_col = "%s_cold" % self.fields.itemid
        self.test = _Test(None, pd.DataFrame({self.fields.userid: cold_user[keep_row][order],
                                              cold_col: cold_item[keep_row][order],
                                              self.fields.feedback: cold_fdbk[keep_row][order]}))
        cold_ids = np.flatnonzero(keep_item)
        self.item_features = f
        self.cold_item_features = fc[cold_ids]
        self.representative_users = representative_users
        self.index = _Index(np.arange(n_users), _ItemColdIndex(np.arange(self._train[2][1]), cold_ids), None)
        self.warm_start = False
        self.holdout_size = -1
        self.test_sample = None
        self.train_csr = None
        self.test_csr = None
        self._subscribers = []

    def subscribe(self, event, callback):
        self._subscribers.append((event, callback))

    def to_coo(self, tensor_mode=False, feedback_threshold=None):
        idx, val, shp = self._train
        if tensor_mode:
            raise ValueError("ColdStartData holds 2-way training indices")
        if feedback_threshold is not None:
            keep = val >= feedback_threshold          # data.py:783-788 (filter_values=True)
            idx, val = idx[keep], val[keep]
        return idx.astype(np.intp, copy=False), np.ascontiguousarray(val), shp


# ------------------------------------------------------------------ metrics -------
Hits = namedtuple("Hits", "true_positive false_positive true_negative false_negative")
Relevance = namedtuple("Relevance", "precision recall fallout specifity miss_rate")
Ranking = namedtuple("Ranking", "ndcg ndcl map arhr")
Experience = namedtuple("Experience", "coverage")


def _match_holdout(recs, h_user, h_item):
    """rank (1-based) at which each holdout row appears in its user's list, 0 = absent.  Negative entries (the -1 pads
    of lists shorter than k) are no recommendation, as in build_rank_matrix (evaluation.py:29-36)."""
    m, k = recs.shape
    n_items = int(max(recs.max(), h_item.max())) + 1
    rec_key = (np.repeat(np.arange(m, dtype=np.int64), k) * n_items + recs.ravel().astype(np.int64))
    rec_key[recs.ravel() < 0] = -1
    order = np.argsort(rec_key, kind="stable")
    sorted_key = rec_key[order]
    hold_key = h_user.astype(np.int64) * n_items + h_item.astype(np.int64)
    pos = np.searchsorted(sorted_key, hold_key)
    pos = np.minimum(pos, len(sorted_key) - 1)
    found = sorted_key[pos] == hold_key
    rank = np.zeros(len(hold_key), dtype=np.int64)
    rank[found] = (order[pos[found]] % k) + 1
    return rank


def _safe_mean_ratio(num, den, mask):
    out = np.zeros(num.shape, dtype=np.float64)
    np.divide(num, den, out=out, where=mask)
    return out.mean()


HitRate = namedtuple("Relevance", "hr")
ReciprocalRank = namedtuple("Ranking", "arhr mrr")


def evaluate_lists(recs, h_user, h_item, h_fdbk, n_items_total, metric_type="all", switch_positive=None,
                   not_rated_penalty=None, ndcg_alternative=True, simple_rates=False):
    """Metrics of polara/recommender/evaluation.py:90-253 computed from ``[m x k]`` lists and
    the holdout triplets (users 0..m-1, sorted).  Masked divisions yield 0 (the reference's
    ``safe_divide``, evaluation.py:18-20, leaves such entries uninitialised)."""
    if metric_type == "all":
        metric_type = ["hits", "relevance", "ranking", "experience"]
    elif metric_type == "main":
        metric_type = ["relevance", "ranking"]
    elif not isinstance(metric_type, (list, tuple)):
        metric_type = [metric_type]
    recs = np.asarray(recs)
    m, k = recs.shape
    # rows of ``recs`` are aligned with the sorted unique holdout users
    # (matrix_from_observations, evaluation.py:45-62, cuts rows at np.diff(keys))
    h_user = np.unique(np.asarray(h_user), return_inverse=True)[1].astype(np.int64)
    h_item = np.asarray(h_item)
    rank = _match_holdout(recs, h_user, h_item)
    if switch_positive is None or h_fdbk is None:
        penalty = 1 if not_rated_penalty is None else not_rated_penalty      # models.py:431-437
        positive = np.ones(len(rank), dtype=bool)
        has_neg = False
    else:
        penalty = not_rated_penalty or 0                                      # models.py:438-444
        positive = np.asarray(h_fdbk) >= switch_positive
        has_neg = True
    hit = rank > 0
    per_user = lambda mask: np.bincount(h_user[mask], minlength=m).astype(np.float64)  # noqa: E731
    tp = per_user(hit & positive)
    n_pos = per_user(positive)
    fn = n_pos - tp
    n_valid = (recs >= 0).sum(axis=1).astype(np.float64)
    if has_neg:
        fp = per_user(hit & ~positive)
        tn = per_user(~positive) - fp
        if penalty > 0:
            fp = fp + penalty * (n_valid - tp - fp)
    else:
        fp = penalty * (n_valid - tp) if penalty > 0 else np.zeros(m)
        tn = None
    scores = []
    if simple_rates:
        # models.py:451-452, 457-458 (holdout_size == 1 or simple_rates): hit rate and reciprocal ranks of the positive
        # hits only (evaluation.py:101-118)
        hp = hit & positive
        if "relevance" in metric_type:
            scores.append(HitRate(tp.mean()))
        if "ranking" in metric_type:
            inv = np.zeros(len(rank), dtype=np.float64)
            inv[hp] = 1.0 / rank[hp]
            arhr = np.bincount(h_user[hp], weights=inv[hp], minlength=m).mean()
            best = np.zeros(m, dtype=np.float64)
            np.maximum.at(best, h_user[hp], inv[hp])
            scores.append(ReciprocalRank(arhr, best.mean()))
        metric_type = [t for t in metric_type if t not in ("relevance", "ranking")]
    if "relevance" in metric_type:
        precision = _safe_mean_ratio(tp, tp + fp, tp > 0)
        recall = _safe_mean_ratio(tp, tp + fn, tp > 0)
        miss_rate = _safe_mean_ratio(fn, fn + tp, fn > 0)
        if tn is not None:
            fallout = _safe_mean_ratio(fp, fp + tn, fp > 0)
            specifity = _safe_mean_ratio(tn, fp + tn, tn > 0)
        else:
            fallout = specifity = None
        scores.append(Relevance(precision, recall, fallout, specifity, miss_rate))
    if "ranking" in metric_type:
        fd = np.ones(len(rank)) if h_fdbk is None else np.asarray(h_fdbk, dtype=np.float64)

        def ndcr(values, sel, sign):
            rel = np.exp2(values) - 1 if ndcg_alternative else values        # evaluation.py:155-158
            disc = np.zeros(len(rank))
            disc[hit] = 1.0 / np.log2(1.0 + rank[hit])
            dcr = np.bincount(h_user[sel], weights=(rel * disc * sign)[sel], minlength=m)
            # ideal: each user's holdout sorted by feedback descending gets 1/log2(2..)
            order = np.lexsort((-fd, h_user))
            starts = np.r_[0, np.flatnonzero(np.diff(h_user[order])) + 1]
            within = np.arange(len(order)) - np.repeat(starts, np.diff(np.r_[starts, len(order)]))
            ideal = np.empty(len(rank))
            ideal[order] = 1.0 / np.log2(2.0 + within)
            idcr = np.bincount(h_user[sel], weights=(rel * ideal * sign)[sel], minlength=m)
            return _safe_mean_ratio(dcr, idcr, dcr > 0)

        ndcg = ndcr(fd, positive, 1.0)
        ndcl = ndcr(fd - switch_positive, ~positive, -1.0) if has_neg else None
        hp = hit & positive
        arhr = np.bincount(h_user[hp], weights=1.0 / rank[hp], minlength=m).mean()
        # MAP (evaluation.py:120-133): precision at each hit position / min(#relevant, k)
        ap = np.zeros(m)
        if hp.any():
            order = np.lexsort((rank[hp], h_user[hp]))
            uu, rr = h_user[hp][order], rank[hp][order]
            starts = np.r_[0, np.flatnonzero(np.diff(uu)) + 1]
            nth = np.arange(len(uu)) - np.repeat(starts, np.diff(np.r_[starts, len(uu)])) + 1
            ap = np.bincount(uu, weights=nth / rr, minlength=m)
        n_rel = np.bincount(h_user, minlength=m)
        ap = ap / np.where(n_rel < k, np.maximum(n_rel, 1), k)
        scores.append(Ranking(ndcg, ndcl, ap.mean(), arhr))
    if "experience" in metric_type:
        scores.append(Experience(len(np.unique(recs)) / n_items_total))
    if "hits" in metric_type:
        scores.append(Hits(int(tp.sum()), fp.sum() if np.ndim(fp) else fp,
                           None if tn is None else int(tn.sum()), int(fn.sum())))
    if not scores:
        raise NotImplementedError
    return scores[0] if len(scores) == 1 else scores


# ------------------------------------------------------------- model base ---------
class RecommenderModel:
    """Mirror of polara/recommender/models.py:71-604 restricted to what the hot path uses."""

    _config = ("topk", "filter_seen", "switch_positive", "feedback_threshold", "verify_integrity")
    _pad_const = -1

    def __init__(self, recommender_data, feedback_threshold=None):
        self.data = recommender_data
        self._recommendations = None
        self.method = "ABC"
        self._topk = DEFAULTS["topk"]
        self._filter_seen = DEFAULTS["filter_seen"]
        self._feedback_threshold = feedback_threshold or DEFAULTS["feedback_threshold"]
        self.switch_positive = DEFAULTS["switch_positive"]
        self.verify_integrity = DEFAULTS["verify_integrity"]
        self.max_test_workers = DEFAULTS["max_test_workers"]
        self._prediction_key = self.data.fields.userid
        self._prediction_target = self.data.fields.itemid
        self._is_ready = False
        self.verbose = True
        self.training_time = []
        self.data.subscribe(self.data.on_change_event, self._renew_model)
        self.data.subscribe(self.data.on_update_event, self._refresh_model)

    def __init_subclass__(cls, **kw):
        # MetaModel (models.py:59-67): any subclass ``build`` resets the cached state
        super().__init_subclass__(**kw)
        if "build" in cls.__dict__:
            inner = cls.__dict__["build"]

            def build(self, *args, _inner=inner, **kwargs):
                self._is_ready = False
                self._recommendations = None
                res = _inner(self, *args, **kwargs)
                self._is_ready = True
                return res
            build.__doc__ = inner.__doc__
            build.__wrapped__ = inner
            cls.build = build

    @property
    def recommendations(self):                                   # models.py:100-108
        if self._recommendations is None:
            if not self._is_ready:
                if self.verbose:
                    print("{} model is not ready. Rebuilding.".format(self.method))
                self.build()
            self._recommendations = self.get_recommendations()
        return self._recommendations

    def _renew_model(self):
        self._recommendations = None
        self._is_ready = False

    def _refresh_model(self):
        self._recommendations = None

    @property
    def topk(self):
        return self._topk

    @topk.setter
    def topk(self, new_value):                                   # models.py:123-128
        if (self._recommendations is not None) and (new_value > self._recommendations.shape[1]):
            self._recommendations = None
        self._topk = new_value

    @property
    def feedback_threshold(self):
        return self._feedback_threshold

    @feedback_threshold.setter
    def feedback_threshold(self, new_value):
        if self._feedback_threshold != new_value:
            self._feedback_threshold = new_value
            self._renew_model()

    @property
    def filter_seen(self):
        return self._filter_seen

    @filter_seen.setter
    def filter_seen(self, new_value):
        if self._filter_seen != new_value:
            self._filter_seen = new_value
            self._refresh_model()

    def build(self):
        raise NotImplementedError("This must be implemented in subclasses")

    def _get_test_data(self, feedback_threshold=None):           # models.py:227-257
        try:
            tensor_mode = self.factors.get(self.data.fields.feedback, None) is not None
        except AttributeError:
            tensor_mode = False
        test_shape = self.data.get_test_shape(tensor_mode=tensor_mode)
        threshold = feedback_threshold or self.feedback_threshold
        if self.data.warm_start:
            if threshold:
                print("Specifying threshold has no effect in warm start.")
            threshold = None
        user_idx, item_idx, feedback = self.data.test_to_coo(tensor_mode=tensor_mode, feedback_threshold=threshold)
        idx_diff = np.diff(user_idx)
        assert (idx_diff >= 0).all()  # calculations assume testset is sorted by users!
        if (idx_diff > 1).any() or (user_idx.min() != 0):
            test_users = user_idx[np.r_[0, np.where(idx_diff)[0] + 1]]
            user_idx = np.r_[0, np.cumsum(idx_diff > 0)].astype(user_idx.dtype)
        else:
            test_users = np.arange(test_shape[0])
        return (user_idx, item_idx, feedback), test_shape, test_users

    def get_recommendations(self):
        raise NotImplementedError("This must be implemented in subclasses")

    # ---- the two hooks of the reference's chunk driver, kept callable for FOREIGN dense scores ------------------------
    # (our own models never materialise score rows: pb200_score_topk fuses contraction, masking and top-k)
    @staticmethod
    def _dense_block(scores):
        import scipy.sparse as sps
        import torch
        if sps.issparse(scores):
            raise NotImplementedError("sparse score matrices (models.py:501-509, 524-560) are not on the device path")
        if isinstance(scores, torch.Tensor):
            return scores, None
        arr = np.asarray(scores)
        if arr.dtype not in (np.float32, np.float64):
            arr = arr.astype(np.float64)
        return None, np.ascontiguousarray(arr) if arr.ndim == 2 else np.ascontiguousarray(arr.reshape(1, -1))

    @staticmethod
    def downvote_seen_items(recs, idx_seen):
        """models.py:494-519, dense branch, IN PLACE: seen scores move below the block minimum, order preserved.
        ``recs``: numpy [m x n] (float32/float64) or a CUDA tensor; ``idx_seen``: (user_idx, item_idx[, ...])."""
        from .engine import get_engine
        import torch
        eng = get_engine()
        dev, host = RecommenderModel._dense_block(recs)
        rows = np.asarray(idx_seen[0]).astype(np.int64, copy=False)
        cols = np.asarray(idx_seen[1]).astype(np.int64, copy=False)
        if host is not None and np.ndim(recs) == 1:
            rows = np.zeros(len(cols), dtype=np.int64)      # single-user form (models.py:513-515)
        block = dev if dev is not None else eng.upload(host)
        eng.downvote_dense(block, eng.upload(rows), eng.upload(cols))
        if dev is None:
            np.asarray(recs).reshape(host.shape)[...] = block.cpu().numpy()

    def get_topk_elements(self, scores):
        """models.py:522-564, dense branch: ``[rows x topk]`` item ids by descending score (ties: smaller id first)."""
        eng = getattr(self, "engine", None)
        if eng is None:
            from .engine import get_engine
            eng = get_engine()
        dev, host = self._dense_block(scores)
        block = dev if dev is not None else eng.upload(host)
        if self.topk > block.shape[1]:
            raise ValueError("topk exceeds the number of items")       # np.argpartition raises, models.py:490
        return eng.topk_dense(block, self.topk).cpu().numpy()

    def evaluate(self, metric_type="all", topk=None, not_rated_penalty=None, switch_positive=None,
                 ignore_feedback=False, simple_rates=False, on_feedback_level=None):
        """models.py:408-485."""
        if int(topk or 0) > self.topk:
            self.topk = topk
        recommendations = self.recommendations[:, :topk]
        switch_positive = switch_positive or self.switch_positive
        f = self.data.fields
        holdout = self.data.test.holdout
        # assemble_scoring_matrices (models.py:445-446): lists are matched by the holdout's key and target columns --
        # (user, item) pairs, or (cold item, user) pairs in item cold start
        h_user = np.asarray(holdout[self._prediction_key].values, dtype=np.int64)
        h_item = np.asarray(holdout[self._prediction_target].values, dtype=np.int64)
        h_fdbk = None if (f.feedback is None or ignore_feedback) else np.asarray(holdout[f.feedback].values)
        if f.feedback is None:
            switch_positive = None
        fd_for_pos = None if f.feedback is None else np.asarray(holdout[f.feedback].values)
        res = evaluate_lists(recommendations, h_user, h_item,
                             fd_for_pos if h_fdbk is None and switch_positive is not None else h_fdbk,
                             self._target_entity_count(), metric_type=metric_type,
                             switch_positive=switch_positive, not_rated_penalty=not_rated_penalty,
                             ndcg_alternative=DEFAULTS["ndcg_alternative"],
                             simple_rates=simple_rates or getattr(self.data, "holdout_size", None) == 1)
        return res

    def _target_entity_count(self):
        """the coverage denominator (models.py:465-471): the size of the index of the entity the lists hold -- items, or
        the training users in item cold start.  A target that is not a field (the holdout positions of sampled
        evaluation) counts the items."""
        fields = self.data.fields
        target = self._prediction_target if self._prediction_target in fields else fields.itemid
        entity_index = getattr(self.data.index, fields._fields[fields.index(target)])
        try:
            return entity_index.shape[0]
        except AttributeError:
            return entity_index.training.shape[0]
