"""Known answers of the reference's window tests (dask_sql tests/integration/test_over.py), transcribed as data:
name -> (table, columns of the table, query, expected output columns in the table's row order)."""
USER_TABLE_1 = {"user_id": [2, 1, 2, 3], "b": [3, 3, 1, 3]}
USER_TABLE_2 = {"user_id": [1, 1, 2, 4], "c": [1, 2, 3, 4]}

CASES = {
    "over_with_partitioning": (
        "user_table_2", USER_TABLE_2,
        'SELECT user_id, c, ROW_NUMBER() OVER (PARTITION BY c) AS "R" FROM user_table_2',
        {"R": [1, 1, 1, 1]}),
    "over_with_grouping_and_sort": (
        "user_table_1", USER_TABLE_1,
        'SELECT user_id, b, ROW_NUMBER() OVER (PARTITION BY user_id ORDER BY b) AS "R" FROM user_table_1',
        {"R": [2, 1, 1, 1]}),
    "over_with_different": (
        "user_table_1", USER_TABLE_1,
        'SELECT user_id, b, ROW_NUMBER() OVER (PARTITION BY user_id ORDER BY b) AS "R1", '
        'ROW_NUMBER() OVER (ORDER BY user_id, b) AS "R2" FROM user_table_1',
        {"R1": [2, 1, 1, 1], "R2": [3, 1, 2, 4]}),
    "over_calls": (
        "user_table_1", USER_TABLE_1,
        'SELECT user_id, b, ROW_NUMBER() OVER (PARTITION BY user_id ORDER BY b) AS "O1", '
        'FIRST_VALUE(user_id*10 - b) OVER (PARTITION BY user_id ORDER BY b) AS "O2", '
        'LAST_VALUE(user_id*10 - b) OVER (PARTITION BY user_id ORDER BY b ROWS BETWEEN UNBOUNDED PRECEDING AND '
        'UNBOUNDED FOLLOWING) AS "O4", SUM(user_id) OVER (PARTITION BY user_id ORDER BY b) AS "O5", '
        'AVG(user_id) OVER (PARTITION BY user_id ORDER BY b) AS "O6", '
        'COUNT(*) OVER (PARTITION BY user_id ORDER BY b) AS "O7", COUNT(b) OVER (PARTITION BY user_id ORDER BY b) '
        'AS "O7b", MAX(b) OVER (PARTITION BY user_id ORDER BY b) AS "O8", '
        'MIN(b) OVER (PARTITION BY user_id ORDER BY b) AS "O9" FROM user_table_1',
        {"O1": [2, 1, 1, 1], "O2": [19, 7, 19, 27], "O4": [17, 7, 17, 27], "O5": [4, 1, 2, 3],
         "O6": [2, 1, 2, 3], "O7": [2, 1, 1, 1], "O7b": [2, 1, 1, 1], "O8": [3, 3, 1, 3], "O9": [1, 3, 1, 3]}),
    "over_with_windows": (
        "tmp", {"a": [0, 1, 2, 3, 4]},
        'SELECT a, '
        'SUM(a) OVER (ORDER BY a ROWS BETWEEN 2 PRECEDING AND CURRENT ROW) AS "O1", '
        'SUM(a) OVER (ORDER BY a ROWS BETWEEN 2 PRECEDING AND 3 FOLLOWING) AS "O2", '
        'SUM(a) OVER (ORDER BY a ROWS BETWEEN 2 PRECEDING AND UNBOUNDED FOLLOWING) AS "O3", '
        'SUM(a) OVER (ORDER BY a ROWS BETWEEN CURRENT ROW AND 3 FOLLOWING) AS "O4", '
        'SUM(a) OVER (ORDER BY a ROWS BETWEEN CURRENT ROW AND UNBOUNDED FOLLOWING) AS "O5", '
        'SUM(a) OVER (ORDER BY a ROWS BETWEEN UNBOUNDED PRECEDING AND CURRENT ROW) AS "O6", '
        'SUM(a) OVER (ORDER BY a ROWS BETWEEN UNBOUNDED PRECEDING AND 3 FOLLOWING) AS "O7", '
        'SUM(a) OVER (ORDER BY a ROWS BETWEEN UNBOUNDED PRECEDING AND UNBOUNDED FOLLOWING) AS "O8", '
        'SUM(a) OVER (ORDER BY a ROWS BETWEEN 3 FOLLOWING AND 3 FOLLOWING) AS "O9", '
        'COUNT(a) OVER (ORDER BY a ROWS BETWEEN 3 FOLLOWING AND 3 FOLLOWING) AS "O9a", '
        'SUM(a) OVER (ORDER BY a ROWS BETWEEN 3 PRECEDING AND 1 PRECEDING) AS "O10" FROM tmp',
        {"O1": [0, 1, 3, 6, 9], "O2": [6, 10, 10, 10, 9], "O3": [10, 10, 10, 10, 9], "O4": [6, 10, 9, 7, 4],
         "O5": [10, 10, 9, 7, 4], "O6": [0, 1, 3, 6, 10], "O7": [6, 10, 10, 10, 10], "O8": [10, 10, 10, 10, 10],
         "O9": [3, 4, None, None, None], "O9a": [1, 1, 0, 0, 0], "O10": [None, 0, 1, 3, 6]}),
}
