"""Subqueries in expressions: [NOT] IN (SELECT ...), [NOT] EXISTS (SELECT ...) and (SELECT ...) as a value.

The reference evaluates `x IN (SELECT y ...)` with its operator table's "in subquery" (call.py:996-1030,
InSubqueryOperation: series.isin of the computed column) and runs EXISTS as the LEFTSEMI / LEFTANTI joins
DataFusion decorrelates it into (physical/rel/logical/join.py:46-47, 146-229).  Here both are a mark: before a
Filter or Projection converts its expressions, attach_marks stacks one MarkSource per IN / EXISTS call on the
block's frame (after the Filter's other conjuncts), and the operators "in subquery" and "exists" read the mark
column it added.  A scalar subquery that refers to no outer column runs when the statement is converted and
becomes a literal."""
from collections import OrderedDict

from .... import executor
from ....datacontainer import DataContainer
from ....frame import LazyFrame, MarkSource, is_lazy
from ....utils import new_temporary_column
from ..base import BaseRexPlugin
from ..convert import RexConverter


def _body_frame(plan, context) -> LazyFrame:
    """the subquery body's rows, one column per output field in order (two fields may be the same column)"""
    from ...rel import RelConverter
    dc = RelConverter.convert(plan, context=context)
    frame, cc = dc.df, dc.column_container
    exprs = OrderedDict((f"__sq{k}", frame.exprs[cc.get_backend_by_frontend_name(name)])
                        for k, name in enumerate(cc.columns))
    return LazyFrame(frame.source, exprs, frame.pred)


def attach_marks(rel, rexes, dc: DataContainer, context) -> DataContainer:
    """dc with the mark of every IN / EXISTS call of the expressions `rexes` as a column of its frame, all stacked
    in one pass so that every mark is a column of the returned frame.  dc.marks maps each call's Subquery to its
    column name (uncorrelated EXISTS: to its constant)."""
    calls = [e for rex in rexes for e in rex.subqueries() if e.value.kind != "scalar"]
    if not calls:
        return dc
    frame, cc = dc.df, dc.column_container
    marks = dict(getattr(dc, "marks", None) or {})
    why = executor.mark_refusal(frame)
    if why is not None:
        raise NotImplementedError(why)
    for e in calls:
        sq = e.value
        inner = _body_frame(sq.plan, context)
        why = executor.mark_refusal(inner)
        if why is not None:
            raise NotImplementedError(why)
        if not sq.keys:                              # uncorrelated EXISTS
            marks[id(sq)] = (None, executor.count_rows(inner) > 0)
            continue
        outer = {}
        for a in e.args:
            v = RexConverter.convert(rel, a, DataContainer(frame, cc), context=context)
            if not is_lazy(v):
                raise NotImplementedError(f"a subquery compared with the constant {a.display()}: compare a column")
            outer[new_temporary_column(frame)] = v
        frame = frame.assign(**outer)
        names = list(outer)
        keys = [(names[i], inner.columns[k]) for i, k in enumerate(sq.keys)]
        terms = [(names[len(sq.keys) + t], inner.columns[k], op, where) for t, (k, op, where) in enumerate(sq.terms)]
        column = new_temporary_column(frame)
        marks[id(sq)] = (column, None)
        frame = LazyFrame(MarkSource(frame, inner, keys, terms, sq.null_aware, column))
    out = DataContainer(frame, cc)
    out.marks = marks
    return out


def mark_of(rex, dc):
    """the value of an IN / EXISTS call over dc, whose frame attach_marks gave the call's mark column"""
    marks = getattr(dc, "marks", None) or {}
    if id(rex.value) not in marks:
        raise NotImplementedError(f"{rex.display()}: IN / EXISTS subqueries are supported in WHERE, HAVING and the "
                                  "SELECT list")
    column, constant = marks[id(rex.value)]
    return constant if column is None else dc.df[column]


class ScalarSubqueryPlugin(BaseRexPlugin):
    """(SELECT one_value ...): zero rows are NULL, one row its value, more rows an error."""

    class_name = "ScalarSubquery"

    def convert(self, rel, rex, dc, context):
        inner = _body_frame(rex.value.plan, context)
        if len(inner.columns) != 1:
            raise ValueError(f"a scalar subquery returns one column, not {len(inner.columns)}")
        got = inner.compute()
        if len(got) > 1:
            raise ValueError("scalar subquery returned more than one row")
        if len(got) == 0:
            return None
        v = got.iloc[0, 0]
        if v is None or v != v:
            return None
        return v.item() if hasattr(v, "item") else v
