"""dtype <-> SQL type mapping for the hot-path types (mirrors dask_sql/mappings.py:17-363 for
BIGINT / DOUBLE / BOOLEAN and the narrower numeric types that widen onto them)."""
import numpy as np
import pandas as pd

from . import temporal as T
from .frame import LazyFrame, LazySeries


class SqlTypeName:
    """String-valued stand-in for the Rust enum dask_sql._datafusion_lib.SqlTypeName."""

    _names = ["ANY", "BIGINT", "BOOLEAN", "DOUBLE", "FLOAT", "REAL", "INTEGER", "SMALLINT", "TINYINT",
              "DECIMAL", "NULL", "VARCHAR", "CHAR", "DATE", "TIMESTAMP", "TIME", "INTERVAL"]

    def __init__(self, name):
        self.name = name.upper()

    def __str__(self):
        return f"SqlTypeName.{self.name}"

    __repr__ = __str__

    def __eq__(self, other):
        return isinstance(other, SqlTypeName) and other.name == self.name

    def __hash__(self):
        return hash(self.name)

    @classmethod
    def fromString(cls, s):
        s = str(s).upper().replace("SQLTYPENAME.", "")
        alias = {"INT": "INTEGER", "INT64": "BIGINT", "INT32": "INTEGER", "INT16": "SMALLINT", "INT8": "TINYINT",
                 "FLOAT64": "DOUBLE", "FLOAT32": "FLOAT", "BOOL": "BOOLEAN", "UTF8": "VARCHAR", "STRING": "VARCHAR",
                 "UINT8": "TINYINT", "UINT16": "SMALLINT", "UINT32": "INTEGER", "UINT64": "BIGINT",
                 "DOUBLE PRECISION": "DOUBLE", "TEXT": "VARCHAR"}
        s = alias.get(s, s)
        if s not in cls._names:
            raise NotImplementedError(f"SQL type {s} is not supported by this layer")
        return cls(s)


for _n in SqlTypeName._names:
    setattr(SqlTypeName, _n, SqlTypeName(_n))

_PYTHON_TO_SQL = {
    "float64": SqlTypeName.DOUBLE, "float32": SqlTypeName.FLOAT, "Float64": SqlTypeName.DOUBLE,
    "Float32": SqlTypeName.FLOAT,
    "int64": SqlTypeName.BIGINT, "Int64": SqlTypeName.BIGINT, "int32": SqlTypeName.INTEGER,
    "Int32": SqlTypeName.INTEGER, "int16": SqlTypeName.SMALLINT, "Int16": SqlTypeName.SMALLINT,
    "int8": SqlTypeName.TINYINT, "Int8": SqlTypeName.TINYINT, "uint64": SqlTypeName.BIGINT,
    "UInt64": SqlTypeName.BIGINT, "uint32": SqlTypeName.INTEGER, "UInt32": SqlTypeName.INTEGER,
    "uint16": SqlTypeName.SMALLINT, "UInt16": SqlTypeName.SMALLINT, "uint8": SqlTypeName.TINYINT,
    "UInt8": SqlTypeName.TINYINT, "bool": SqlTypeName.BOOLEAN, "boolean": SqlTypeName.BOOLEAN,
}

_SQL_TO_PYTHON = {
    "DOUBLE": np.float64, "FLOAT": np.float32, "REAL": np.float32, "DECIMAL": np.float64,
    "BIGINT": np.int64, "INTEGER": np.int32, "SMALLINT": np.int16, "TINYINT": np.int8,
    "BOOLEAN": np.bool_, "NULL": type(None),
}


def python_to_sql_type(python_type) -> SqlTypeName:
    """mappings.py:92-116.  datetime64[D] (and date32) is DATE, datetime64[s|ms|us|ns] is TIMESTAMP;
    time-zone-aware and timedelta types are not supported."""
    key = str(python_type)
    if key == "category":             # dictionary-coded strings (strings.py)
        return SqlTypeName.VARCHAR
    sql = T.sql_type_of(key)
    if sql is not None:
        return SqlTypeName(sql)
    try:
        return _PYTHON_TO_SQL[key]
    except KeyError:
        raise NotImplementedError(f"The python type {python_type} is not implemented (yet)")


def sql_to_python_type(sql_type, *args):
    name = sql_type.name if isinstance(sql_type, SqlTypeName) else SqlTypeName.fromString(sql_type).name
    if name == "DATE":
        return np.dtype("datetime64[D]")
    if name == "TIMESTAMP":
        return np.dtype(f"datetime64[{T.DEFAULT_UNIT}]")
    try:
        return _SQL_TO_PYTHON[name]
    except KeyError:
        raise NotImplementedError(f"The SQL type {name} is not implemented (yet)")


def sql_to_python_value(sql_type, literal_value):
    """mappings.py:145-262, numeric/boolean rows."""
    name = sql_type.name if isinstance(sql_type, SqlTypeName) else SqlTypeName.fromString(sql_type).name
    if literal_value is None or name == "NULL":
        return None
    if name in ("DOUBLE", "FLOAT", "REAL", "DECIMAL"):
        return float(literal_value)
    if name in ("BIGINT", "INTEGER", "SMALLINT", "TINYINT"):
        if isinstance(literal_value, T.TScalar):       # CAST(DATE '...' AS BIGINT): its ticks
            return literal_value.ticks
        return int(literal_value)
    if name == "BOOLEAN":
        return bool(literal_value)
    if name in ("VARCHAR", "CHAR"):
        return str(literal_value)
    if name in ("DATE", "TIMESTAMP"):
        # a DATE / TIMESTAMP value, or a string read as one (CAST('1995-03-15' AS DATE))
        if isinstance(literal_value, T.TScalar):
            if name == "DATE":
                return T.TScalar(T.datepart(literal_value.ticks, "DAYS", literal_value.unit), "D")
            return T.TScalar(literal_value.at(T.DEFAULT_UNIT), T.DEFAULT_UNIT) if literal_value.unit == "D" \
                else literal_value
        try:
            return T.parse_date(str(literal_value)) if name == "DATE" else T.parse_timestamp(str(literal_value))
        except ValueError as err:
            from .utils import ParsingException
            raise ParsingException(str(literal_value), str(err)) from None
    if name == "INTERVAL" and isinstance(literal_value, T.Interval):
        return literal_value
    raise NotImplementedError(f"literal of SQL type {name}")


_SIMILAR_CACHE = {}


def similar_type(lhs, rhs) -> bool:
    """Same type family (int / float / bool): no cast needed (mappings.py:264-306)."""
    key = (str(lhs), str(rhs))
    hit = _SIMILAR_CACHE.get(key)
    if hit is not None:
        return hit
    ul, ur = T.unit_of(lhs), T.unit_of(rhs)
    if ul is not None or ur is not None:     # DATE and TIMESTAMP are two families; units do not matter
        out = ul is not None and ur is not None and (ul == "D") == (ur == "D")
        _SIMILAR_CACHE[key] = out
        return out
    pdt = pd.api.types
    l, r = pd.api.types.pandas_dtype(lhs), pd.api.types.pandas_dtype(rhs)
    out = False
    for check in (pdt.is_bool_dtype, pdt.is_integer_dtype, pdt.is_float_dtype):
        if check(l) and check(r):
            out = True
            break
    _SIMILAR_CACHE[key] = out
    return out


def cast_column_type(df: LazyFrame, column_name: str, expected_type) -> LazyFrame:
    """Cast df[column_name] only if its type family differs (mappings.py:309-329)."""
    current = df.dtype_of(column_name)
    if expected_type is type(None) or similar_type(current, expected_type):
        return df
    casted = cast_column_to_type(df[column_name], expected_type)
    if casted is None:
        return df
    return df.assign(**{column_name: casted})


def cast_column_to_type(col: LazySeries, expected_type):
    """mappings.py:332-363: float -> int casts truncate (da.trunc) first; no-op returns None."""
    if similar_type(col.dtype, expected_type):
        return None
    return col.astype(np.dtype(expected_type) if expected_type is not np.bool_ else "bool")
