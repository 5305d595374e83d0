"""The reference's known answers for its numeric functions, TRANSCRIBED from dask-contrib/dask-sql @ f186de3,
tests/integration/test_rex.py:488-545 (test_math_operations), over the `df` fixture of reference_vectors.py
(tests/integration/fixtures.py:50-57).  SELECT lists each column with its alias; EXPECTED is the NumPy / pandas
expression the reference test compares that column with.  Nothing here is produced by our own code."""
import numpy as np

CITE = "tests/integration/test_rex.py:488-545"

SELECT = [
    ("ABS(b)", "abs"), ("ACOS(b)", "acos"), ("ASIN(b)", "asin"), ("ATAN(b)", "atan"), ("ATAN2(a, b)", "atan2"),
    ("CBRT(b)", "cbrt"), ("CEIL(b)", "ceil"), ("COS(b)", "cos"), ("COT(b)", "cot"), ("DEGREES(b)", "degrees"),
    ("EXP(b)", "exp"), ("FLOOR(b)", "floor"), ("LOG10(b)", "log10"), ("LN(b)", "ln"), ("MOD(b, 4)", "mod"),
    ("POWER(b, 2)", "power"), ("POWER(b, a)", "power2"), ("RADIANS(b)", "radians"), ("ROUND(b)", "round"),
    ("ROUND(b, 3)", "round2"), ("SIGN(b)", "sign"), ("SIN(b)", "sin"), ("TAN(b)", "tan"),
    ("TRUNCATE(b)", "truncate"),
]

SQL = "SELECT " + ", ".join(f'{e} AS "{a}"' for e, a in SELECT) + " FROM df"

EXPECTED = {
    "abs": lambda df: df.b.abs(),
    "acos": lambda df: np.arccos(df.b),
    "asin": lambda df: np.arcsin(df.b),
    "atan": lambda df: np.arctan(df.b),
    "atan2": lambda df: np.arctan2(df.a, df.b),
    "cbrt": lambda df: np.cbrt(df.b),
    "ceil": lambda df: np.ceil(df.b),
    "cos": lambda df: np.cos(df.b),
    "cot": lambda df: 1 / np.tan(df.b),
    "degrees": lambda df: df.b / np.pi * 180,
    "exp": lambda df: np.exp(df.b),
    "floor": lambda df: np.floor(df.b),
    "log10": lambda df: np.log10(df.b),
    "ln": lambda df: np.log(df.b),
    "mod": lambda df: np.mod(df.b, 4),
    "power": lambda df: np.power(df.b, 2),
    "power2": lambda df: np.power(df.b, df.a),
    "radians": lambda df: df.b / 180 * np.pi,
    "round": lambda df: np.round(df.b),
    "round2": lambda df: np.round(df.b, 3),
    "sign": lambda df: np.sign(df.b),
    "sin": lambda df: np.sin(df.b),
    "tan": lambda df: np.tan(df.b),
    "truncate": lambda df: np.trunc(df.b),
}
