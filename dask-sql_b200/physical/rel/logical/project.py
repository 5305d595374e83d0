"""Projection (dask_sql/physical/rel/logical/project.py:17-78).

A projected plain column reference costs nothing: the output name is mapped onto the backend
column it already is.  Every other item becomes one lazy expression column under a temporary
backend name; nothing is evaluated here -- the executor fuses the expression into whichever
kernel consumes it."""
from ....datacontainer import DataContainer
from ....planner import RexType
from ....utils import new_temporary_column
from ...rex import RexConverter
from ...rex.core.subquery import attach_marks
from ..base import BaseRelPlugin

_REFERENCE = str(RexType.Reference)


class DaskProjectPlugin(BaseRelPlugin):
    class_name = "Projection"

    def convert(self, rel, context) -> DataContainer:
        (child,) = self.assert_inputs(rel, 1, context)
        child = attach_marks(rel, [expr for _, expr in rel.projection().getNamedProjects()], child, context)
        frame, names = child.df, child.column_container
        computed, backend_of = {}, {}
        for out_name, expr in rel.projection().getNamedProjects():
            if str(expr.getRexType()) == _REFERENCE:
                backend_of[str(out_name)] = names.get_backend_by_frontend_index(expr.getIndex())
            else:
                tmp = new_temporary_column(frame)
                computed[tmp] = RexConverter.convert(rel, expr, child, context=context)
                backend_of[str(out_name)] = tmp
        if computed:
            frame = frame.assign(**computed)
        for out_name, backend in backend_of.items():
            names = names.add(out_name, backend)
        names = self.fix_column_to_row_type(names.limit_to(list(backend_of)), rel.getRowType())
        return self.fix_dtype_to_row_type(DataContainer(frame, names), rel.getRowType())
