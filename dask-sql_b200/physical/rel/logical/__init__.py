"""Plan-node plugins of the filter -> join -> group-by path and the operators either side of it."""
from . import (aggregate, cross_join, empty, explain, filter, join, limit, project, sort,  # noqa: A004
               subquery_alias, table_scan, window)

DaskTableScanPlugin = table_scan.DaskTableScanPlugin
DaskFilterPlugin = filter.DaskFilterPlugin
DaskProjectPlugin = project.DaskProjectPlugin
DaskJoinPlugin = join.DaskJoinPlugin
DaskCrossJoinPlugin = cross_join.DaskCrossJoinPlugin
DaskAggregatePlugin = aggregate.DaskAggregatePlugin
DaskSortPlugin = sort.DaskSortPlugin
DaskLimitPlugin = limit.DaskLimitPlugin
SubqueryAlias = subquery_alias.SubqueryAlias
ExplainPlugin = explain.ExplainPlugin
DaskEmptyRelationPlugin = empty.DaskEmptyRelationPlugin
DaskWindowPlugin = window.DaskWindowPlugin

ALL_PLUGINS = (DaskTableScanPlugin, DaskFilterPlugin, DaskProjectPlugin, DaskJoinPlugin, DaskCrossJoinPlugin,
               DaskAggregatePlugin, DaskSortPlugin, DaskLimitPlugin, SubqueryAlias, ExplainPlugin, DaskEmptyRelationPlugin,
               DaskWindowPlugin)
