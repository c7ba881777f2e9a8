"""Rank search of an SVD model with the lists of every rank computed in one device sweep.

:func:`find_optimal_svd_rank` has the signature and the semantics of ``polara.evaluation.pipelines.find_optimal_svd_rank``
(pipelines.py:81-116): build once at the largest rank, then evaluate the truncated model at each rank, largest first.
The reference recomputes the recommendations at every rank; here they come from one call made before the loop --
``rank_sweep`` for the standard protocol, ``sampled_rank_sweep`` for sampled evaluation -- which shares the test-data
ingest, the SpMM at the largest rank and, on the sampled protocol, the draw of the unseen items between all ranks.  The
evaluator then sees the model at each rank with ``_recommendations`` set to that rank's lists.  Item cold-start models
(users as the target) have a feature transform per rank and take the reference's per-rank loop instead.

:func:`find_optimal_tucker_ranks` does the same for a CoFFee model (pipelines.py:119-160): build once at the largest rank
of each mode, then evaluate every multilinear rank ``(r1, r2, r3)`` of the grid.  The lists of all triples come from one
``tucker_rank_sweep`` made before the loop, which ingests the test data once and rotates only the item factor on the
device.  The evaluator sees ``_mlrank`` set to each triple and ``_recommendations`` set to that triple's lists; unlike
the reference, ``factors`` stay those of the full build, because rounding the user factor is the cost the sweep removes.
"""
from __future__ import annotations

from collections.abc import Iterable, Mapping

from .models import sampled_protocol_inputs

__all__ = ["evaluate_models", "find_optimal_svd_rank", "find_optimal_tucker_ranks", "rank_sweep_lists",
           "set_config"]


def set_config(model, config, convert_nan=True):
    """pipelines.py:56-60: set every ``name: value`` of ``config`` as a model attribute (NaN -> None)."""
    for name, value in config.items():
        if convert_nan and value != value:
            value = None
        setattr(model, name, value)


def evaluate_models(models, target_metric="precision", metric_type="all", **kwargs):
    """pipelines.py:63-78: ``{model.method: target metric}`` of ``model.evaluate(metric_type, **kwargs)`` for one model or
    a collection of them; ``target_metric`` is a metric name or a callable applied to the row of all metrics."""
    import pandas as pd
    if isinstance(models, (str, bytes, Mapping)) or not isinstance(models, Iterable):
        models = [models]
    out = {}
    for model in models:
        res = model.evaluate(metric_type, **kwargs)
        row = pd.concat([pd.DataFrame([r]) for r in (res if isinstance(res, list) else [res])], axis=1)
        if isinstance(target_metric, str):
            value = row[target_metric]
        elif callable(target_metric):
            value = row.apply(target_metric, axis=1)
        else:
            raise NotImplementedError("target_metric must be a metric name or a callable")
        out[model.method] = value.squeeze()
    return out


def rank_sweep_lists(model, ranks):
    """``{rank: lists}`` of ``model.recommendations`` at every rank.  Items as the target: one standard sweep.  Users as
    the target (item cold start): the reference's loop, ``model.rank = r`` then ``get_recommendations()`` with ranks
    descending, because every rank has its own feature transform; the model's rank, factors and transform are restored
    afterwards.  Anything else predicts holdout positions: one sampled sweep, its inputs read from the data model as the
    sampled drop-in's ``get_recommendations`` reads them."""
    fields = model.data.fields
    if model._prediction_target == fields.itemid:
        return model.rank_sweep(ranks)
    if model._prediction_target == fields.userid:
        state = _rank_state(model)
        try:
            lists = {}
            for rank in sorted(set(ranks), reverse=True):
                model.rank = rank
                lists[rank] = model.get_recommendations()
            return lists
        finally:
            _restore_rank_state(model, state)
    holdout_items, unseen, kwargs = sampled_protocol_inputs(model)
    return model.sampled_rank_sweep(ranks, holdout_items, unseen, **kwargs)


def _rank_state(model):
    return model._rank, dict(model.factors), getattr(model, "_item_features_transform_helper", None)


def _restore_rank_state(model, state):
    model._rank, model.factors = state[0], dict(state[1])
    if hasattr(model, "_item_features_transform_helper"):
        model._item_features_transform_helper = state[2]


def find_optimal_svd_rank(model, ranks, target_metric, return_scores=False, protect_factors=True, config=None,
                          verbose=False, evaluator=None, iterator=lambda x: x, **kwargs):
    """pipelines.py:81-116 with the lists of all ranks from one device sweep (see the module docstring).  Returns the
    rank with the best ``target_metric`` and, with ``return_scores``, the Series of scores in the order of ``ranks``.
    ``evaluator(model, target_metric, **kwargs)`` defaults to :func:`evaluate_models`."""
    import pandas as pd
    evaluator = evaluator or evaluate_models
    model_verbose = model.verbose
    if config:
        set_config(model, config)
    svd_rank = max(max(ranks), model.rank)
    model.rank = svd_rank
    if not model._is_ready:
        model.verbose = verbose
        model.build()
    if protect_factors:
        svd_state = _rank_state(model)       # the transform of a cold-start model goes with its factors
    res = {}
    try:
        lists = rank_sweep_lists(model, ranks)
        for rank in iterator(sorted(ranks, reverse=True)):
            model.rank = rank
            model._recommendations = lists[rank]
            res[rank] = evaluator(model, target_metric, **kwargs)[model.method]
            model._recommendations = None          # the next rank must not see this rank's lists
    finally:
        if protect_factors:
            _restore_rank_state(model, svd_state)
        model.verbose = model_verbose
    scores = pd.Series(res)
    best_rank = scores.idxmax()
    if return_scores:
        scores.index.name = "rank"
        scores.name = model.method
        return best_rank, scores.loc[list(ranks)]
    return best_rank


def _tucker_grid(tucker_ranks, same_space=False):
    """The triples pipelines.py:141-148 visits, in its order: ``r1`` of ``tucker_ranks[0]``, ``r2`` of
    ``tucker_ranks[1]`` (only ``r2 == r1`` with ``same_space``), ``r3`` of ``tucker_ranks[2]``, skipping a triple where
    one rank exceeds the product of the other two."""
    return [(r1, r2, r3) for r1 in tucker_ranks[0] for r2 in tucker_ranks[1] if not (same_space and r2 != r1)
            for r3 in tucker_ranks[2] if not (r1 * r2 < r3 or r1 * r3 < r2 or r2 * r3 < r1)]


def find_optimal_tucker_ranks(model, tucker_ranks, target_metric, return_scores=False, config=None, verbose=False,
                              same_space=False, evaluator=None, iterator=lambda x: x, **kwargs):
    """pipelines.py:119-160 with the lists of all triples from one ``tucker_rank_sweep`` (see the module docstring).
    ``model.mlrank`` is set to the largest rank of each mode and the model is built if it is not ready; then
    ``evaluator(model, target_metric, **kwargs)[model.method]`` (default :func:`evaluate_models`) scores each triple of
    the grid, ``iterator`` wrapping the ranks of the first mode as in the reference.  During each call the model
    shows ``_mlrank`` equal to the triple and that triple's lists, but the factors of the full build, not the rounded
    ones.  ``_mlrank`` and ``factors`` are restored afterwards, also when the evaluator raises; ``verbose`` is restored
    after the loop.  Returns the best triple and, with ``return_scores``, the Series of scores indexed by
    ``(r1, r2, r3)``."""
    import pandas as pd
    evaluator = evaluator or evaluate_models
    model_verbose = model.verbose
    if config:
        set_config(model, config)
    model.mlrank = tuple([max(mode_ranks) for mode_ranks in tucker_ranks])
    if not model._is_ready:
        model.verbose = verbose
        model.build()
    factors = dict(**model.factors)
    tucker_rank = model.mlrank
    grid = _tucker_grid(tucker_ranks, same_space)
    res_score = {}
    try:
        lists = model.tucker_rank_sweep(grid) if grid else {}
        for r1 in iterator(tucker_ranks[0]):
            for mlrank in _tucker_grid(([r1],) + tuple(tucker_ranks[1:]), same_space):
                model._mlrank = mlrank
                model._recommendations = lists[mlrank]
                res_score[mlrank] = evaluator(model, target_metric, **kwargs)[model.method]
                model._recommendations = None          # the next triple must not see this triple's lists
    finally:
        model._mlrank = tucker_rank
        model.factors = dict(**factors)
        model._recommendations = None
    model.verbose = model_verbose
    scores = pd.Series(res_score).sort_index()
    best_mlrank = scores.idxmax()
    if return_scores:
        scores.index.names = ["r1", "r2", "r3"]
        scores.name = model.method
        return best_mlrank, scores
    return best_mlrank
