"""Aggregate / Distinct: GROUP BY, global aggregates, DISTINCT (the reference's plugin is
dask_sql/physical/rel/logical/aggregate.py:91-589).

The reference runs one  groupby(keys, dropna=False).agg(...)  per (FILTER column, DISTINCT column)
bucket and stitches the buckets together by index (aggregate.py:334-375, 522-589), with a constant
key column standing in for "no GROUP BY" (aggregate.py:305-306).  Here the node is first described as
a list of AggCall records, then laid out as PASSES over the input:

  * every call without DISTINCT shares ONE pass -- `agg(x) FILTER (WHERE f)` is rewritten to
    `agg(CASE WHEN f THEN x END)`, which every aggregate treats as "skip the row" -- so the common
    query is a single AggSource, i.e. one fused kernel pass at compute time (b2_scan_agg,
    b2_groupby_*, or the star / join-aggregate pipelines when a Join sits underneath);
  * calls with DISTINCT get one pass per distinct input, over the de-duplicated (keys, input) pairs;
  * passes are stitched by a left join on the keys (a literal key when there are none).

STDDEV / VARIANCE are handed to the executor by name: it accumulates shifted moments in the same
pass (executor.AggPlan), not sum-of-squares around zero.
"""
import logging
from collections import OrderedDict
from dataclasses import dataclass
from typing import Optional

from .... import config as dask_config
from ....datacontainer import ColumnContainer, DataContainer
from ....frame import AggSource, LazyFrame, LazySeries
from ....expr import ColRef
from ....utils import new_temporary_column
from ...rex.convert import RexConverter
from ..base import BaseRelPlugin

logger = logging.getLogger(__name__)

# SQL aggregate name -> the executor's name for it (aggregate.py:117-231 lists the reference's table;
# these are its hot-path rows).  "sum" means sum(min_count=1): an all-NULL group sums to NULL.
_EXECUTOR_NAME = {
    "sum": "sum", "$sum0": "sum", "avg": "mean", "mean": "mean", "count": "count", "min": "min", "max": "max",
    "stddev": "stddev_samp", "stddev_samp": "stddev_samp", "stddevsamp": "stddev_samp",
    "stddev_pop": "stddev_pop", "stddevpop": "stddev_pop",
    "variance": "var_samp", "var_samp": "var_samp", "var": "var_samp",
    "var_pop": "var_pop", "variance_pop": "var_pop", "variancepop": "var_pop",
    "bit_and": "bit_and", "bit_or": "bit_or", "bit_xor": "bit_xor", "every": "every",
    "regr_count": "count", "regr_sxx": "regr_sxx", "regr_syy": "regr_syy",
}
# REGR_*(y, x): the one aggregate family with two inputs.  Only rows where BOTH are non-NULL count, so the
# input is  x' = CASE WHEN y IS NOT NULL THEN x END  (y' likewise for REGR_SYY), and REGR_COUNT is COUNT(x').
_REGR = {"regr_count": 1, "regr_sxx": 1, "regr_syy": 0}   # which argument is aggregated


@dataclass
class AggCall:
    out: str                          # output column = the plan's rendering of the call
    fn: str                           # executor function name
    arg: Optional[LazySeries]         # input values, None for COUNT(*)
    keep: Optional[LazySeries]        # FILTER (WHERE ...) condition
    distinct: bool


class DaskAggregatePlugin(BaseRelPlugin):
    class_name = ["Aggregate", "Distinct"]

    def convert(self, rel, context) -> DataContainer:
        (child,) = self.assert_inputs(rel, 1, context)
        node = rel.aggregate()
        names = child.column_container.make_unique()
        frame = child.df
        if node.isDistinctNode():
            key_fields = list(node.getDistinctColumns())
        else:
            key_fields = [g.column_name(rel) for g in node.getGroupSets()]
        keys = [names.get_backend_by_frontend_name(k) for k in key_fields]
        calls = self._describe(rel, node, DataContainer(frame, names), context)
        options = dask_config.get("sql.aggregate") or {}
        if calls:
            result = self._run_passes(frame, keys, calls, options)
        else:
            result = frame[keys].drop_duplicates(**options)          # DISTINCT / GROUP BY without aggregates
        shown = ColumnContainer(result.columns).limit_to(keys + [c.out for c in calls])
        shown = self.fix_column_to_row_type(shown, rel.getRowType())
        return self.fix_dtype_to_row_type(DataContainer(result, shown), rel.getRowType())

    # -- 1. what the node asks for ---------------------------------------------------------------
    def _describe(self, rel, node, child: DataContainer, context):
        input_rel = rel.get_inputs()[0]
        known = child.column_container

        def value_of(rex) -> LazySeries:
            field = rex.column_name(input_rel)
            if known.knows(field):             # a plain input column
                return child.df[known.get_backend_by_frontend_name(field)]
            return RexConverter.convert(input_rel, rex, child, context=context)

        calls = []
        for call in node.getNamedAggCalls():
            assert call.getExprType() in {"Alias", "AggregateFunction", "AggregateUDF"}, \
                f"unexpected aggregate expression {call.getExprType()}"
            sql_name = node.getAggregationFuncName(call).lower()
            if sql_name not in _EXECUTOR_NAME:
                raise NotImplementedError(f"Aggregation function {sql_name} not implemented (yet).")
            args = node.getArgs(call)
            if sql_name in _REGR:
                vals = [value_of(a) for a in args]
                if not all(isinstance(v, LazySeries) for v in vals):
                    raise NotImplementedError(f"{sql_name.upper()} over a literal argument")
                i = _REGR[sql_name]
                arg = vals[i].where(vals[1 - i].notna())
            elif len(args) > 1:
                raise NotImplementedError("aggregates over more than one input column")
            else:
                arg = value_of(args[0]) if args else None
            if arg is None and call.isDistinctAgg():
                raise NotImplementedError("COUNT(DISTINCT *)")
            keep = call.getFilterExpr()
            calls.append(AggCall(call.toString(), _EXECUTOR_NAME[sql_name] if arg is not None else "size", arg,
                                 value_of(keep) if keep is not None else None, bool(call.isDistinctAgg())))
        return calls

    # -- 2. passes over the input ----------------------------------------------------------------
    @staticmethod
    def _column_for(frame: LazyFrame, series: LazySeries):
        """(frame, column name) holding `series`: the input column itself when it is one, else a fresh
        computed column (still lazy: it fuses into the aggregation kernel's scan)."""
        e = series.expr
        for name, have in frame.exprs.items():
            if have is e or (isinstance(e, ColRef) and isinstance(have, ColRef) and have.name == e.name):
                return frame, name
        name = new_temporary_column(frame)
        return frame.assign(**{name: series}), name

    def _run_passes(self, frame, keys, calls, options):
        shared, per_distinct_input = [], OrderedDict()
        for c in calls:
            fn, values = c.fn, c.arg
            if values is not None and not isinstance(values, LazySeries):
                # a literal argument (SUM(2), COUNT(1)): a constant column of the input
                name = new_temporary_column(frame)
                frame = frame.assign(**{name: values})
                values = frame[name]
            if c.keep is not None:
                if values is None:                                    # COUNT(*) FILTER (WHERE f) = COUNT(f or NULL)
                    fn, values = "count", c.keep.where(c.keep)
                else:
                    values = values.where(c.keep)
            column = None
            if values is not None:
                frame, column = self._column_for(frame, values)
            if c.distinct:
                per_distinct_input.setdefault(column, []).append((column, c.out, fn))
            else:
                shared.append((column, c.out, fn))
        passes = []
        if shared:
            passes.append((frame, shared))
        for column, specs in per_distinct_input.items():
            passes.append((frame.drop_duplicates(subset=keys + [column], **options), specs))
        logger.debug("aggregate: %d pass(es) over the input", len(passes))

        join_keys = keys
        if len(passes) > 1 and not keys:
            # global aggregates from several passes: each pass yields one row; give them a literal key
            # to meet on (the reference's constant-column trick, aggregate.py:305-306)
            one = new_temporary_column(frame)
            passes = [(f.assign(**{one: 0}), specs) for f, specs in passes]
            join_keys = [one]
        result = None
        for source, specs in passes:
            part = LazyFrame(AggSource(source, join_keys, specs, options))
            if result is None:
                result = part
                continue
            # the first pass holds every group (it saw every row); later ones hang off it
            theirs = {k: f"{k}__pass{len(result.columns)}" for k in join_keys}
            merged = result.merge(part.rename(theirs), how="left", left_on=join_keys,
                                  right_on=[theirs[k] for k in join_keys])
            result = merged[list(result.columns) + [out for _, out, _ in specs]]
        return result if join_keys is keys else result[[c for c in result.columns if c not in join_keys]]
