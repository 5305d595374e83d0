"""The reference's EXISTS test, transcribed as data: tests/integration/test_rex.py:570-587 (test_subqueries,
xfail there: "Subquery expressions not yet enabled") over the fixtures user_table_1 / user_table_2
(tests/integration/fixtures.py:66-72).  Its intended answer is user_table_2[user_table_2.c.isin(user_table_1.b)]."""

USER_TABLE_1 = {"user_id": [2, 1, 2, 3], "b": [3, 3, 1, 3]}
USER_TABLE_2 = {"user_id": [1, 1, 2, 4], "c": [1, 2, 3, 4]}

EXISTS_SQL = """
    SELECT *
    FROM
        user_table_2
    WHERE
        EXISTS(
            SELECT *
            FROM user_table_1
            WHERE
                user_table_1.b = user_table_2.c
        )
"""

# (user_id, c) rows of the answer, in the fixture's order
EXISTS_ANSWER = [(1, 1), (2, 3)]
