"""Literal -> python value (dask_sql/physical/rex/core/literal.py:82-201, numeric/boolean rows)."""
from ....mappings import SqlTypeName, sql_to_python_value
from ..base import BaseRexPlugin

_ARROW_TO_SQL = {
    "Boolean": ("BOOLEAN", "getBoolValue"), "Float32": ("FLOAT", "getFloat32Value"),
    "Float64": ("DOUBLE", "getFloat64Value"), "Int8": ("TINYINT", "getInt8Value"),
    "Int16": ("SMALLINT", "getInt16Value"), "Int32": ("INTEGER", "getInt32Value"),
    "Int64": ("BIGINT", "getInt64Value"), "UInt8": ("TINYINT", "getUInt8Value"),
    "UInt16": ("SMALLINT", "getUInt16Value"), "UInt32": ("INTEGER", "getUInt32Value"),
    "UInt64": ("BIGINT", "getUInt64Value"), "Utf8": ("VARCHAR", "getStringValue"),
    "Date32": ("DATE", "getTemporalValue"), "Timestamp": ("TIMESTAMP", "getTemporalValue"),
    "IntervalMonthDayNano": ("INTERVAL", "getTemporalValue"),
}


class RexLiteralPlugin(BaseRexPlugin):
    class_name = "RexLiteral"

    def convert(self, rel, rex, dc, context):
        literal_type = str(rex.getType())
        if literal_type == "Null":
            return None
        try:
            sql_name, getter = _ARROW_TO_SQL[literal_type]
        except KeyError:
            raise RuntimeError(f"Failed to map literal type {literal_type} to python type in literal.py")
        try:
            value = getattr(rex, getter)()
        except TypeError:
            return None  # NULL boolean literal (literal.py:103-108)
        return sql_to_python_value(SqlTypeName.fromString(sql_name), value)
