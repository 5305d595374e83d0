"""Context: the public API object (mirrors dask_sql/context.py:51-983 for the hot-path surface:
create_table / drop_table / sql / explain / register of plugins, schemas, config_options).

    from dask_sql_b200 import Context
    c = Context()
    c.create_table("t", pandas_df, persist=True)        # columns -> HBM (Arrow layout)
    c.sql("SELECT SUM(x) FROM t WHERE x > 0").compute()  # -> pandas.DataFrame
"""
import logging
import warnings
from collections import Counter
from typing import Any, Dict, Optional, Union

import pandas as pd
import torch

from . import config as dask_config
from .datacontainer import ColumnContainer, DataContainer, SchemaContainer, Statistics
from .frame import LazyFrame, TableSource
from .mappings import python_to_sql_type
from .physical.rel import RelConverter
from .physical.rel import custom, logical
from .physical.rex import RexConverter
from .physical.rex import core
from .planner import LogicalPlan, plan_sql
from .table import DeviceTable
from .utils import OptimizationException, ParsingException

logger = logging.getLogger(__name__)


class Context:
    """Holds registered tables and turns SQL into lazy device frames.

    Plugins are registered with replace=False (context.py:118-158) so a plugin registered
    earlier — or later with replace=True — wins: that is the drop-in seam."""

    DEFAULT_CATALOG_NAME = "dask_sql"
    DEFAULT_SCHEMA_NAME = "root"

    def __init__(self, logging_level=logging.INFO, device: Optional[int] = None):
        self.catalog_name = self.DEFAULT_CATALOG_NAME
        self.schema_name = self.DEFAULT_SCHEMA_NAME
        self.schema: Dict[str, SchemaContainer] = {self.schema_name: SchemaContainer(self.schema_name)}
        self.device = device
        self.sql_server = None
        self._catalog_version = 0          # bumped by create_table / drop_table / schema changes
        self._plan_cache = {}
        logger.setLevel(logging_level)

        # replace=False: whoever registered a plugin for a node type before us -- or registers one
        # later with replace=True -- wins (context.py:118-158); that is the drop-in seam
        for plugin in (*logical.ALL_PLUGINS, custom.CreateMemoryTablePlugin, custom.CreateTablePlugin,
                       custom.DropTablePlugin, custom.AnalyzeTablePlugin):
            RelConverter.add_plugin_class(plugin, replace=False)
        for plugin in core.ALL_PLUGINS:
            RexConverter.add_plugin_class(plugin, replace=False)

    # -- catalog ------------------------------------------------------------------------------
    def _torch_device(self):
        if not torch.cuda.is_available():
            raise RuntimeError("dask_sql_b200 executes on a CUDA device (H100, sm_90a); no CPU fallback exists")
        return torch.device("cuda", self.device if self.device is not None else torch.cuda.current_device())

    def create_table(self, table_name: str, input_table: Any, format: str = None, persist: bool = False,
                     schema_name: str = None, statistics: Statistics = None, gpu: bool = False, **kwargs):
        """Register a table (context.py:168-293).

        input_table: pandas.DataFrame, dict of column -> numpy array / torch tensor, pyarrow.Table,
        a DeviceTable, a LazyFrame (e.g. the result of another query), or the path of a Parquet /
        CSV file (format = "parquet" | "csv", default by extension; kwargs `columns=[...]` reads a subset).
        persist=True uploads the columns to HBM once; persist=False (the reference's default:
        'the data will be lazily loaded') keeps them in pinned host memory and streams them to the
        GPU for every query.  kwargs: npartitions (default 1, pandaslike.py:26) and
        distribution = 'local' | 'sharded' | 'replicated' | 'root' for multi-GPU jobs.

        VARCHAR columns are stored as int64 codes into a sorted per-column dictionary.  They come from
        input that is already dictionary-typed -- a pandas `category` column with string categories, an
        Arrow `dictionary<int*, string>` column (chunks may carry different dictionaries), a Parquet
        column read back as one -- or from `dictionary=["col", ...]`, which dictionary-encodes the named
        plain string columns of any input (Parquet: read_dictionary, CSV: a dictionary column type).
        Any other string column raises NotImplementedError.  VARCHAR results come back as `category`.
        A VARCHAR column cannot be in a 'sharded' or 'root' table: each rank would build its own
        dictionary."""
        logger.debug(f"Creating table: '{table_name}' of format type '{format}' in schema '{schema_name}'")
        schema_name = schema_name or self.schema_name
        npartitions = kwargs.pop("npartitions", 1)
        distribution = kwargs.pop("distribution", "local")
        dictionary = list(kwargs.pop("dictionary", None) or ())
        filepath = None
        if isinstance(input_table, str) and not persist:
            import os
            from .table import ParquetTable, location_format
            if location_format(input_table, format) == "parquet" and os.path.isfile(input_table):
                # persist=False ('the data will be lazily loaded'): row groups become partitions, read per
                # query and pruned by the pushed-down filters (table_scan.py:80-99, physical/utils/filter.py)
                kwargs.pop("gpu", None)
                filepath = input_table
                input_table = ParquetTable(input_table, distribution, table_name, kwargs.pop("columns", None),
                                           dictionary)
                if kwargs:
                    raise TypeError(f"unsupported options for reading {filepath!r}: {sorted(kwargs)}")
        if isinstance(input_table, LazyFrame):
            df = input_table.persist() if persist else input_table
        else:
            if isinstance(input_table, DeviceTable):
                table = input_table
            else:
                if isinstance(input_table, str):
                    # storage location (input_utils/location.py:11-54): Parquet / CSV column chunks are
                    # read with pyarrow and laid out on the device without a pandas detour
                    from .table import read_location
                    input_table = read_location(input_table, format, dictionary=dictionary, **kwargs)
                    kwargs = {}
                if type(input_table).__module__.startswith("pyarrow") and hasattr(input_table, "column_names"):
                    from .table import arrow_columns
                    columns = arrow_columns(input_table, dictionary)  # pyarrow.Table: buffers used as they are
                elif isinstance(input_table, pd.DataFrame):
                    columns = {str(c): input_table[c] for c in input_table.columns}
                elif isinstance(input_table, dict):
                    columns = {str(k): v for k, v in input_table.items()}
                else:
                    raise NotImplementedError(f"cannot create a table from {type(input_table).__name__}")
                for name in dictionary:
                    if name not in columns:
                        raise KeyError(f"dictionary=: no column {name!r}")
                    if not hasattr(columns[name], "logical"):
                        columns[name] = pd.Series(columns[name]).astype("category")
                dev = self._torch_device() if persist else None
                table = DeviceTable.from_columns(columns, npartitions, dev, persist, distribution, table_name)
            table.name = table_name
            df = LazyFrame(TableSource(table))
        dc = DataContainer(df, ColumnContainer(df.columns))
        dc.view = isinstance(input_table, LazyFrame) and not persist    # no row numbers to sample by
        if not statistics:
            statistics = Statistics(float("nan"))
        dc.statistics = statistics
        dc.filepath = filepath
        self.schema[schema_name].tables[table_name.lower()] = dc
        self.schema[schema_name].statistics[table_name.lower()] = statistics
        if filepath is not None:
            self.schema[schema_name].filepaths[table_name.lower()] = filepath
        self._catalog_version += 1

    def drop_table(self, table_name: str, schema_name: str = None):
        schema_name = schema_name or self.schema_name
        del self.schema[schema_name].tables[table_name.lower()]
        self._catalog_version += 1

    def create_schema(self, schema_name: str):
        self.schema[schema_name] = SchemaContainer(schema_name)
        self._catalog_version += 1

    def drop_schema(self, schema_name: str):
        if schema_name == self.DEFAULT_SCHEMA_NAME:
            raise RuntimeError(f"Default Schema `{schema_name}` cannot be deleted")
        del self.schema[schema_name]
        self._catalog_version += 1
        if self.schema_name == schema_name:
            self.schema_name = self.DEFAULT_SCHEMA_NAME

    def fqn(self, tbl) -> tuple:
        """(schema, table) of a plan's table reference (context.py:731-747)."""
        schema_name = tbl.getSchema()
        if schema_name is None or schema_name == "":
            schema_name = self.schema_name
        return schema_name, tbl.getTableName()

    # -- queries ------------------------------------------------------------------------------
    def sql(self, sql: Any, return_futures: bool = True, dataframes: Dict[str, Any] = None, gpu: bool = False,
            config_options: Dict[str, Any] = None) -> Union[LazyFrame, pd.DataFrame]:
        """Run a SELECT (context.py:482-533).  return_futures=True gives the lazy frame
        (.compute() executes it); False computes and returns a pandas DataFrame."""
        with dask_config.set(config_options):
            if dataframes is not None:
                for df_name, df in dataframes.items():
                    self.create_table(df_name, df, gpu=gpu)
            if isinstance(sql, str):
                # prepared-statement cache: planning + plugin conversion are pure functions of
                # (SQL text, catalog, config), and LazyFrames are immutable
                from .utils import Pluggable
                key = (sql, self._catalog_version, Pluggable.version, self.schema_name, dask_config.get("sql.optimize"),
                       dask_config.get("sql.identifier.case_sensitive"), dask_config.get("sql.join.broadcast"),
                       str(dask_config.get("sql.aggregate")))
                df = self._plan_cache.get(key)
                if df is None:
                    rel, _ = self._get_ral(sql)
                    df = self._compute_table_from_rel(rel, True)
                    if isinstance(df, LazyFrame) and not getattr(rel, "volatile", False):
                        if len(self._plan_cache) > 256:
                            self._plan_cache.clear()
                        self._plan_cache[key] = df
                if return_futures or not isinstance(df, LazyFrame):
                    return df
                return df.compute()
            elif isinstance(sql, LogicalPlan):
                rel = sql
            else:
                raise RuntimeError(f"Encountered unsupported `LogicalPlan` sql type: {type(sql)}")
            return self._compute_table_from_rel(rel, return_futures)

    def explain(self, sql: str, dataframes: Dict[str, Any] = None, gpu: bool = False) -> str:
        """The optimised relational algebra as text (context.py:535-571)."""
        if dataframes is not None:
            for df_name, df in dataframes.items():
                self.create_table(df_name, df, gpu=gpu)
        _, rel_string = self._get_ral(sql)
        return rel_string

    def _catalog(self, schema_name: Optional[str], table_name: str):
        schema_name = schema_name or self.schema_name
        container = self.schema.get(schema_name)
        if container is None:
            return None
        dc = container.tables.get(table_name.lower())
        if dc is None:
            return None
        cols = []
        dtypes = dc.df.dtypes
        for frontend, backend in zip(dc.column_container.columns,
                                     [dc.column_container.get_backend_by_frontend_name(c)
                                      for c in dc.column_container.columns]):
            cols.append((frontend, python_to_sql_type(dtypes[backend]).name))
        return schema_name, cols

    def _get_ral(self, sql):
        """SQL -> (optimised plan, explain string) (context.py:819-872)."""
        logger.debug(f"Entering _get_ral('{sql}')")
        case_sensitive = dask_config.get("sql.identifier.case_sensitive")
        rel = None
        if dask_config.get("sql.optimize"):
            try:
                rel = plan_sql(sql, self._catalog, case_sensitive, optimize_plan=True)
            except ParsingException:
                raise
            except Exception as e:  # optimizer failure -> unoptimised plan (context.py:858-864)
                warnings.warn(f"The optimizer failed ({OptimizationException(e)}); using the unoptimized plan")
        if rel is None:
            rel = plan_sql(sql, self._catalog, case_sensitive, optimize_plan=False)
        rel_string = rel.explain_original()
        logger.debug(f"_get_ral -> LogicalPlan:\n{rel_string}")
        return rel, rel_string

    def _compute_table_from_rel(self, rel, return_futures: bool = True):
        dc = RelConverter.convert(rel, context=self)
        if rel.get_current_node_type() in ("Explain", "AnalyzeTable"):
            return dc      # the plan text / the statistics frame, already on the host
        if dc is None:
            return
        # keep alias projects; FQ name only where the simple name is ambiguous (context.py:882-906)
        select_names = list(rel.getRowType().getFieldList())
        if select_names:
            cc = dc.column_container
            select_names = select_names[: len(cc.columns)]
            field_counts = Counter([field.getName() for field in select_names])
            select_names = [field.getQualifiedName() if field_counts[field.getName()] > 1 else field.getName()
                            for field in select_names]
            cc = cc.rename({df_col: select_name for df_col, select_name in zip(cc.columns, select_names)})
            dc = DataContainer(dc.df, cc)
        df = dc.assign()
        if not return_futures:
            df = df.compute()
        return df
