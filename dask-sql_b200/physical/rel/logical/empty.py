"""EmptyRelation (dask_sql/physical/rel/logical/empty.py): the input of a SELECT without FROM.

The reference gives such a SELECT a one-row frame with the column `_empty`; here it is a one-row table, so its
row is row 0 of a table and RAND / RAND_INTEGER draw for it as for any table row."""
import numpy as np

from ....datacontainer import ColumnContainer, DataContainer
from ..base import BaseRelPlugin


class DaskEmptyRelationPlugin(BaseRelPlugin):
    class_name = "EmptyRelation"

    def convert(self, rel, context) -> DataContainer:
        from ....frame import LazyFrame, TableSource
        from ....table import DeviceTable
        table = DeviceTable.from_columns({"_empty": np.zeros(1, dtype=np.int64)}, persist=False)
        return DataContainer(LazyFrame(TableSource(table)), ColumnContainer(["_empty"]))
