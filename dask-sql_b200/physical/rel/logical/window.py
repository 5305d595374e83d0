"""Window (dask_sql/physical/rel/logical/window.py): f(...) OVER (PARTITION BY ... ORDER BY ... frame).

The reference sorts each group and applies pandas rolling / expanding per function.  Here the keys and
arguments become columns of the input frame (lazy expressions, evaluated by b2_expr_eval), and one
WindowSource runs every (PARTITION BY, ORDER BY) spec of the node: one sort per spec, shared by its
functions (executor.run_window).  The output keeps the input's rows in their order, with one column per
window call appended."""
from .... import executor
from ....datacontainer import DataContainer
from ....frame import LazyFrame, WindowSource
from ....utils import new_temporary_column
from ...rex.convert import RexConverter
from ..base import BaseRelPlugin


class DaskWindowPlugin(BaseRelPlugin):
    class_name = "Window"

    def convert(self, rel, context) -> DataContainer:
        (dc,) = self.assert_inputs(rel, 1, context)
        frame, cc = dc.df, dc.column_container
        why = executor.window_refusal(frame)
        if why is not None:
            raise NotImplementedError(why)
        node = rel.window()
        input_rel = rel.get_inputs()[0]
        computed = {}

        def column_of(rex) -> str:
            name = rex.column_name(input_rel)
            if cc.knows(name):
                return cc.get_backend_by_frontend_name(name)
            key = rex.display()
            if key not in computed:
                tmp = new_temporary_column(frame)
                computed[key] = (tmp, RexConverter.convert(input_rel, rex, dc, context=context))
            return computed[key][0]

        specs, outputs = [], []
        for _, calls in node.getGroups():
            first = calls[0]
            partition = [column_of(p) for p in node.getPartitionExprs(first)]
            order = [(column_of(s.getSortExpr()), s.isSortAscending(), s.isSortNullsFirst())
                     for s in node.getSortExprs(first)]
            funcs = []
            for call in calls:
                args = node.getArgs(call)
                out = new_temporary_column(frame)
                funcs.append((out, node.getWindowFuncName(call).lower(), column_of(args[0]) if args else None,
                              node.getWindowFrame(call)))
                outputs.append((call.display(), out))
            specs.append((partition, order, funcs))
        if computed:
            frame = frame.assign(**{tmp: value for tmp, value in computed.values()})
        result = LazyFrame(WindowSource(frame, specs))
        by_display = dict(outputs)
        for e in node.window_exprs:
            cc = cc.add(e.display(), by_display[e.display()])
        cc = self.fix_column_to_row_type(cc, rel.getRowType())
        return self.fix_dtype_to_row_type(DataContainer(result, cc), rel.getRowType())
