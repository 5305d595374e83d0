"""ANALYZE TABLE <t> COMPUTE STATISTICS FOR [ALL COLUMNS | COLUMNS a, b, ...]
(dask_sql/physical/rel/custom/analyze_table.py)."""
from collections import OrderedDict

import numpy as np
import pandas as pd

from .... import _lib as L
from .... import strings as S
from .... import temporal as T
from ....expr import ColRef
from ....frame import AggSource, LazyFrame, TableSource
from ....mappings import python_to_sql_type
from ..base import BaseRelPlugin

INDEX = ["count", "mean", "std", "min", "25%", "50%", "75%", "max", "data_type", "col_name"]
QUANTILES = (0.25, 0.5, 0.75)


def _plain_table(df: LazyFrame) -> bool:
    return isinstance(df.source, TableSource) and not df.pred and \
        all(isinstance(e, ColRef) and e.name == n for n, e in df.exprs.items())


def _host_time(ticks, unit):
    """int64 ticks of a DATE / TIMESTAMP column -> the datetime64 array compute() returns for them"""
    return T.to_host_array(np.asarray(ticks, dtype=np.int64), unit)


class AnalyzeTablePlugin(BaseRelPlugin):
    """count, mean, std, min, 25 / 50 / 75 % and max of every analysed column as pandas describe() gives them,
    then its SQL type and name, as a host DataFrame (the reference concatenates describe() with those two rows).

    count, min and max come from the cached column statistics; mean and std from fused global AVG /
    STDDEV_SAMP passes, as many columns to a pass as its accumulators hold (over the int64 ticks of a DATE /
    TIMESTAMP column, whose std stays NaN as in describe()); the quantiles from the two exact order statistics
    around each one (executor.column_quantiles, a GPU radix select), interpolated by pandas itself so that every
    dtype rounds as describe() rounds.  BOOLEAN and VARCHAR columns keep NaN statistics."""

    class_name = "AnalyzeTable"

    def convert(self, rel, context) -> pd.DataFrame:
        from ....executor import column_quantiles

        stmt = rel.analyze_table()
        schema_name = stmt.getSchemaName() or context.schema_name
        dc = context.schema[schema_name].tables[stmt.getTableName()]
        columns = stmt.getColumns() or dc.column_container.columns
        mapping = dc.column_container.get_backend_by_frontend_name
        dtypes = dc.df.dtypes
        df = dc.df if _plain_table(dc.df) else dc.df.persist()
        table = df.source.table

        kind, unit = {}, {}
        for col in columns:
            b = mapping(col)
            dt, lg = df.source.schema[b]
            if dt == L.U8 or S.is_varchar(lg):
                kind[col] = "other"
            elif T.is_temporal(lg):
                kind[col], unit[col] = "time", T.unit_of(lg)
            else:
                kind[col] = "number"

        # mean / std: global aggregates over the described columns (temporal ones as their ticks), as few passes
        # as the accumulators allow: AVG takes one, STDDEV_SAMP at most two more, and a global pass keeps one
        # for its COUNT(*)
        described = [c for c in columns if kind[c] != "other"]
        chunks, slots = [[]], 0
        for col in described:
            need = 3 if kind[col] == "number" else 1
            if slots + need > L.MAX_AGGS - 1:
                chunks, slots = chunks + [[]], 0
            chunks[-1].append(col)
            slots += need
        moments = {}
        for chunk in chunks:
            if not chunk:
                continue
            exprs = OrderedDict()
            aggs = []
            for col in chunk:
                b = mapping(col)
                dt, lg = df.source.schema[b]
                exprs[b] = ColRef(b, dt, "int64" if kind[col] == "time" else lg)
                aggs.append((b, f"mean:{b}", "mean"))
                if kind[col] == "number":
                    aggs.append((b, f"std:{b}", "stddev_samp"))
            res = LazyFrame(AggSource(LazyFrame(TableSource(table), exprs), [], aggs)).compute()
            row = {k: (float(v) if not pd.isna(v) else np.nan) for k, v in zip(res.columns, res.iloc[0])} \
                if len(res) else {}
            for col in chunk:
                b = mapping(col)
                moments[col] = (row.get(f"mean:{b}", np.nan), row.get(f"std:{b}", np.nan))

        out = OrderedDict()
        for col in described + [c for c in columns if kind[c] == "other"]:
            b = mapping(col)
            stats = [np.nan] * 8
            if kind[col] != "other":
                count, vmin, vmax, qs = column_quantiles(table, b, QUANTILES)
                mean, std = moments[col]
                if kind[col] == "number":
                    np_dtype = np.int64 if df.source.schema[b][0] == L.I64 else np.float64
                    stats[0] = float(count)
                    if count:
                        stats[1:3] = [mean, std]
                        stats[3], stats[7] = float(vmin), float(vmax)
                        stats[4:7] = [pd.Series([lo, hi], dtype=np_dtype).quantile(g) for lo, hi, g in qs]
                else:
                    u = unit[col]
                    stats[0] = int(count)
                    if count:
                        host = _host_time([vmin, vmax], u)
                        hu = np.datetime_data(host.dtype)[0]
                        # pandas takes the mean of the host values as float64 and truncates it to a tick
                        per = T.ticks_per_day(hu) if u == "D" else 1
                        stats[1] = pd.Timestamp(np.int64(mean * per).view(f"M8[{hu}]"))
                        stats[3], stats[7] = pd.Timestamp(host[0]), pd.Timestamp(host[1])
                        stats[4:7] = [pd.Series(_host_time([lo, hi], u)).quantile(g) for lo, hi, g in qs]
            out[col] = stats + [str(python_to_sql_type(dtypes[b])).lower(), col]
        return pd.DataFrame(out, index=INDEX, dtype=object)

