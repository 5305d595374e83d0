"""TableScan (dask_sql/physical/rel/logical/table_scan.py:21-119): the registered table, narrowed by
the predicates and the column list the optimizer pushed into the scan.

Nothing is read here.  The pushed-down conjuncts end up as `pred` of the lazy frame and the column
list as its `exprs`, so the kernel that finally consumes the scan evaluates the predicate on the
fly and touches only the columns it needs."""
from ....datacontainer import DataContainer
from ...rex import RexConverter
from ..base import BaseRelPlugin
from .filter import filter_or_scalar


class DaskTableScanPlugin(BaseRelPlugin):
    class_name = "TableScan"

    def convert(self, rel, context) -> DataContainer:
        self.assert_inputs(rel, 0)
        scan, table = rel.table_scan(), rel.getTable()
        schema, name = context.fqn(table)
        registered = context.schema[schema.lower()].tables[name.lower()]
        if scan.sample is not None:
            registered = self._apply_sample(registered, scan.sample, name)
        # predicates before projection: a filter column need not survive into the output
        # (table_scan.py:51-52)
        narrowed = self._apply_projections(scan, table, self._apply_filters(scan, rel, registered, context))
        names = self.fix_column_to_row_type(narrowed.column_container, rel.getRowType())
        return self.fix_dtype_to_row_type(DataContainer(narrowed.df, names), rel.getRowType())

    @staticmethod
    def _apply_sample(dc, sample, name) -> DataContainer:
        """TABLESAMPLE (the reference's physical/rel/logical/sample.py): SYSTEM keeps whole partitions and is
        applied where the table's partitions are read; BERNOULLI puts its row mask in front of every conjunct,
        so each kernel that scans the table filters by it."""
        from ....expr import ColRef, U8
        from ....frame import LazyFrame, TableSource, SAMPLE_MASK
        df = dc.df
        if getattr(dc, "view", False) or not isinstance(df.source, TableSource) or df.pred:
            raise NotImplementedError(f"TABLESAMPLE of the view {name}: only the rows of a base table have numbers "
                                      "to sample by")
        pred = [ColRef(SAMPLE_MASK, U8)] if sample.method == "bernoulli" else []
        frame = LazyFrame(TableSource(df.source.table, sample), type(df.exprs)(df.exprs), pred)
        return DataContainer(frame, dc.column_container)

    def _apply_filters(self, table_scan, rel, dc, context) -> DataContainer:
        """AND of every pushed-down condition (table_scan.py:101-119)."""
        conditions = [RexConverter.convert(rel, rex, dc, context=context) for rex in table_scan.getFilters()]
        if not conditions:
            return dc
        combined = conditions[0]
        for cond in conditions[1:]:
            combined = combined & cond
        return DataContainer(filter_or_scalar(dc.df, combined), dc.column_container)

    def _apply_projections(self, table_scan, dask_table, dc) -> DataContainer:
        """Column subset of the scan, or all of the table's fields (table_scan.py:80-99)."""
        frame, names = dc.df, dc.column_container
        if table_scan.containsProjections():
            keep = [names.get_backend_by_frontend_name(c) for c in table_scan.getTableScanProjects()]
            frame = frame[keep]
        else:
            keep = [str(f).rpartition(".")[2] for f in dask_table.getRowType().getFieldNames()]
        return DataContainer(frame, names.limit_to(keep))
