"""Join: ON clause -> equality key pairs + residual predicate; hash join on the pairs; residual
applied to the join's output (what the reference does in dask_sql/physical/rel/logical/join.py:50-187;
its key extraction is :250-322 and its NULL-key handling + merge :189-248).

Nothing runs here.  The merge is recorded as a JoinSource of the lazy frame; at compute time it becomes
b2_join_build(_dense) + a probe kernel (NULL keys find no partner inside the kernels, which yields the
rows the reference gets by dropping them first), or -- under an Aggregate -- one of the fused
pipelines (b2_star_agg, b2_join_agg) that never materialise the join at all.
"""
import logging

from .... import config as dask_config
from ....datacontainer import ColumnContainer, DataContainer
from ....utils import is_frame
from ...rex import RexConverter
from ..base import BaseRelPlugin
from .filter import filter_or_scalar

logger = logging.getLogger(__name__)

_HOW = {"INNER": "inner", "LEFT": "left", "RIGHT": "right", "FULL": "outer",
        "LEFTSEMI": "leftsemi", "LEFTANTI": "leftanti"}
_LEFT_ONLY_OUTPUT = ("leftsemi", "leftanti")


def _kind(rex) -> str:
    return str(rex.getRexType()).rsplit(".", 1)[-1]


def conjuncts_of(condition):
    """The AND-ed parts of an ON clause, in source order (AND nests arbitrarily in the plan)."""
    parts, todo = [], [condition]
    while todo:
        rex = todo.pop()
        if _kind(rex) == "Call" and str(rex.getOperatorName()).upper() == "AND":
            todo.extend(reversed(list(rex.getOperands())))
        else:
            parts.append(rex)
    return parts


def key_pair(rex, n_left: int):
    """(position in the left input, position in the right input) when `rex` equates one plain column
    of each input, else None.  The plan numbers the join's columns left input first, so a reference
    belongs to the right input iff its index is >= n_left."""
    if _kind(rex) != "Call" or str(rex.getOperatorName()) != "=":
        return None
    operands = list(rex.getOperands())
    if len(operands) != 2 or any(_kind(o) != "Reference" for o in operands):
        return None
    lo, hi = sorted(int(o.getIndex()) for o in operands)
    return (lo, hi - n_left) if lo < n_left <= hi else None


def split_on_clause(condition, n_left: int):
    """-> ([(left pos, right pos), ...], [residual rex, ...])"""
    pairs, residual = [], []
    for part in ([] if condition is None else conjuncts_of(condition)):
        pair = key_pair(part, n_left)
        if pair is None:
            residual.append(part)
        else:
            pairs.append(pair)
    return pairs, residual


def _conjunction(terms):
    """AND of converted residual terms; scalar terms fold with SQL's three-valued logic."""
    verdict, series = True, None
    for t in terms:
        if is_frame(t):
            series = t if series is None else series & t
        elif t is None:
            verdict = None if verdict is True else verdict
        elif not t:
            verdict = False
    if series is None or verdict is not True:
        return verdict               # filter_or_scalar: FALSE / NULL keep nothing, TRUE keeps all
    return series


def _same_unit_keys(left, right, left_on, right_on):
    """DATE / TIMESTAMP keys of different units meet at the finer one: the coarser side joins on a
    scaled copy of its key column (the shown columns stay the inputs' own)."""
    from .... import temporal as T
    from ....utils import new_temporary_column

    left_on, right_on = list(left_on), list(right_on)
    for i, (a, b) in enumerate(zip(left_on, right_on)):
        ua, ub = T.unit_of(left.col_type(a)[1]), T.unit_of(right.col_type(b)[1])
        if ua is None or ub is None or ua == ub:
            continue
        u = T.finer(ua, ub)
        if ua != u:
            name = new_temporary_column(left)
            left = left.assign(**{name: left[a]._wrap(T.at_unit(left[a].expr, u))})
            left_on[i] = name
        else:
            name = new_temporary_column(right)
            right = right.assign(**{name: right[b]._wrap(T.at_unit(right[b].expr, u))})
            right_on[i] = name
    return left, right, left_on, right_on


class DaskJoinPlugin(BaseRelPlugin):
    class_name = "Join"

    def convert(self, rel, context) -> DataContainer:
        node = rel.join()
        left_in, right_in = self.assert_inputs(rel, 2, context)
        how = _HOW[str(node.getJoinType())]
        # both inputs under collision-free backend names, in their SQL column order
        left = DataContainer(left_in.df, left_in.column_container.make_unique("lhs")).assign()
        right = DataContainer(right_in.df, right_in.column_container.make_unique("rhs")).assign()

        pairs, residual = split_on_clause(node.getCondition(), len(left.columns))
        if not pairs:
            raise NotImplementedError(
                "joins without an equality key (cross joins) are outside the hash-join hot path of this layer")
        shown = list(left.columns) + ([] if how in _LEFT_ONLY_OUTPUT else list(right.columns))
        left_on, right_on = [left.columns[i] for i, _ in pairs], [right.columns[j] for _, j in pairs]
        left, right, left_on, right_on = _same_unit_keys(left, right, left_on, right_on)
        joined = left.merge(right, how=how, broadcast=dask_config.get("sql.join.broadcast"),
                            left_on=left_on, right_on=right_on)

        row_type = rel.getRowType()
        names = self.fix_column_to_row_type(ColumnContainer(joined.columns).limit_to(shown), row_type, how)
        out = DataContainer(joined, names)
        if residual:
            keep = _conjunction([RexConverter.convert(rel, rex, out, context=context) for rex in residual])
            logger.debug("residual ON-clause filter: %s", keep)
            out = DataContainer(filter_or_scalar(joined, keep), names)
        return self.fix_dtype_to_row_type(out, row_type, how)
