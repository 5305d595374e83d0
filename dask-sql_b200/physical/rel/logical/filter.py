"""WHERE / HAVING that was not pushed into a scan (dask_sql/physical/rel/logical/filter.py:20-74)."""
import logging

import numpy as np

from ....datacontainer import DataContainer
from ....planner.plan import conjunction, conjuncts
from ...rex import RexConverter
from ...rex.core.subquery import attach_marks
from ..base import BaseRelPlugin

log = logging.getLogger(__name__)


def filter_or_scalar(df, filter_condition, add_filters=None):
    """Rows of `df` for which the condition holds (filter.py:20-45).

    A literal condition keeps everything (truthy) or nothing (falsy / NULL); in a column condition
    NULL counts as False.  On a lazy frame `df[cond]` only records the conjuncts: they run inside the
    consuming kernel as b2_scan_t terms, and only what is not `column <cmp> literal` shaped is
    evaluated as a mask first."""
    if filter_condition is None or (np.isscalar(filter_condition) and not filter_condition):
        if filter_condition is not None:
            log.warning("Join condition is always false - returning empty dataset")
        return df.head(0, compute=False)
    if np.isscalar(filter_condition):
        return df
    return df[filter_condition.fillna(False)]


class DaskFilterPlugin(BaseRelPlugin):
    class_name = "Filter"

    def convert(self, rel, context) -> DataContainer:
        (child,) = self.assert_inputs(rel, 1, context)
        cond = rel.filter().getCondition()
        if cond.contains_subquery():
            # the block's other conjuncts first, so that an IN / EXISTS mark is built over the rows they keep
            plain = [c for c in conjuncts(cond) if not c.contains_subquery()]
            if plain:
                first = conjunction(plain).with_inputs(cond.inputs)
                rest = conjunction([c for c in conjuncts(cond) if c.contains_subquery()]).with_inputs(cond.inputs)
                keep = RexConverter.convert(rel, first, child, context=context)
                child = DataContainer(filter_or_scalar(child.df, keep), child.column_container)
                cond = rest
            child = attach_marks(rel, [cond], child, context)
        keep = RexConverter.convert(rel, cond, child, context=context)
        names = self.fix_column_to_row_type(child.column_container, rel.getRowType())
        return DataContainer(filter_or_scalar(child.df, keep), names)
