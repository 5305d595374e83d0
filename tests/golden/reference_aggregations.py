"""Golden vectors of the reference's test_aggregations (dask-contrib/dask-sql @ f186de3,
tests/integration/test_groupby.py:205-261): EVERY / BIT_AND / BIT_OR next to MIN / AVG, transcribed like the
cases of tests/golden/reference_vectors.py, whose fixtures they use.  The reference's queries also select
SINGLE_VALUE(b), pandas' `first`: it depends on row order, which this layer leaves unspecified, so that
column is left out."""
import pandas as pd

CASES = [
    dict(name="aggregations_every_bit", cite="tests/integration/test_groupby.py:205-232", tables=["user_table_1"],
         sql="SELECT user_id, EVERY(b = 3) AS e, BIT_AND(b) AS b, BIT_OR(b) AS bb, MIN(b) AS m, AVG(b) AS a "
             "FROM user_table_1 GROUP BY user_id",
         expected=pd.DataFrame({"user_id": [1, 2, 3], "e": [True, False, True], "b": [3, 1, 3], "bb": [3, 3, 3],
                                "m": [3, 1, 3], "a": [3.0, 2.0, 3.0]}), float_cols=["a"]),
    dict(name="aggregations_every_bit_2", cite="tests/integration/test_groupby.py:234-261", tables=["user_table_2"],
         sql="SELECT user_id, EVERY(c = 3) AS e, BIT_AND(c) AS b, BIT_OR(c) AS bb, MIN(c) AS m, AVG(c) AS a "
             "FROM user_table_2 GROUP BY user_id",
         expected=pd.DataFrame({"user_id": [1, 2, 4], "e": [False, True, False], "b": [0, 3, 4], "bb": [3, 3, 4],
                                "m": [1, 3, 4], "a": [1.5, 3.0, 4.0]}), float_cols=["a"]),
]
