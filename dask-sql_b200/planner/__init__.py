"""SQL -> optimised logical plan for the hot-path grammar (stand-in for the reference's Rust
planner crate, which needs rustc/cargo and cannot be built in this image; see DESIGN.md)."""
from . import plan  # noqa: F401
from .builder import Binder
from .optimizer import optimize
from .plan import LogicalPlan, PyExpr, RexType, bind_all  # noqa: F401
from .sqlparse import parse_sql


def plan_sql(sql, catalog, case_sensitive=True, optimize_plan=True) -> LogicalPlan:
    tree = parse_sql(sql)
    binder = Binder(sql, catalog, case_sensitive)
    p = binder.bind_statement(tree)
    p = optimize(p) if optimize_plan else bind_all(p)
    p.volatile = binder.volatile      # RAND / TABLESAMPLE without a seed: a new key every time it is planned
    return p
