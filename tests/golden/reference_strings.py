"""Known answers of the reference's string tests, transcribed as data (rows and expected row positions).

string_table: tests/integration/fixtures.py:91-101.  LIKE / ILIKE / NOT / ESCAPE / SIMILAR TO cases:
tests/integration/test_rex.py:255-349; equality filters: tests/integration/test_filter.py:62-73; sort:
tests/integration/test_sort.py:280-295.  `rows` are positions in STRING_TABLE of the expected result;
SIMILAR TO is out of scope here, so its cases are listed with the rows the reference returns and are
expected to raise."""

STRING_TABLE = [
    "a normal string",
    "%_%",
    "^|()-*[]$",
    "^|()-*[]$\n%_%\na normal string",
]

# (predicate over column a, expected row positions)
LIKE_CASES = [
    ("a LIKE '%n[a-z]rmal st_i%'", []),
    ("a NOT LIKE '%n[a-z]rmal st_i%'", [0, 1, 2, 3]),
    ("a LIKE '%a Normal String%'", []),
    ("a ILIKE '%a Normal String%'", [0, 3]),
    ("a NOT ILIKE '%a Normal String%'", [1, 2]),
    ("a LIKE '^|()-*r[r]$' ESCAPE 'r'", [2]),
    ("a LIKE '%_' ESCAPE 'r'", [0, 1, 2, 3]),
]

SIMILAR_CASES = [
    ("a SIMILAR TO '%n[a-z]rmal st_i%'", [0, 3]),
    ("a NOT SIMILAR TO '%n[a-z]rmal st_i%'", [1, 2]),
    ("a SIMILAR TO '^|()-*r[r]$' ESCAPE 'r'", [2, 3]),
]

FILTER_CASES = [
    ("a = 'a normal string'", [0]),
    ("a = 'M'", []),
]

SORT_TABLE = ["zzhsd", "öfjdf", "baba"]
SORT_ASC = ["baba", "zzhsd", "öfjdf"]
