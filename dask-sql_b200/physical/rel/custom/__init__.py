"""Statements around the path: CREATE TABLE ... WITH / AS, CREATE VIEW ... AS, DROP TABLE, ANALYZE TABLE
(dask_sql/physical/rel/custom/)."""
from .analyze_table import AnalyzeTablePlugin
from .create_memory_table import CreateMemoryTablePlugin
from .create_table import CreateTablePlugin
from .drop_table import DropTablePlugin

__all__ = [AnalyzeTablePlugin, CreateMemoryTablePlugin, CreateTablePlugin, DropTablePlugin]
