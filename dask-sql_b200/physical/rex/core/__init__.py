"""Expression plugins of the hot path: calls (operators), column references, literals, aliases."""
from . import alias, call, input_ref, literal, subquery

RexAliasPlugin = alias.RexAliasPlugin
RexCallPlugin = call.RexCallPlugin
RexInputRefPlugin = input_ref.RexInputRefPlugin
RexLiteralPlugin = literal.RexLiteralPlugin
ScalarSubqueryPlugin = subquery.ScalarSubqueryPlugin

ALL_PLUGINS = (RexCallPlugin, RexInputRefPlugin, RexLiteralPlugin, RexAliasPlugin, ScalarSubqueryPlugin)
__all__ = ["RexAliasPlugin", "RexCallPlugin", "RexInputRefPlugin", "RexLiteralPlugin", "ScalarSubqueryPlugin", "ALL_PLUGINS"]
