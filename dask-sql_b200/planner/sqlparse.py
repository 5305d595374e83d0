"""SQL text -> syntax tree for the hot-path grammar.

The reference parses with sqlparser-rs 0.38 inside its Rust crate (src/parser.rs, src/sql.rs:570);
that crate cannot be built here (no rustc/cargo), so this is a small recursive-descent parser for

  [WITH name AS (select) [, ...]]
  SELECT [DISTINCT] item [, ...] FROM source [join ...] [WHERE e] [GROUP BY e, ...] [HAVING e]
  [ORDER BY e [ASC|DESC] [NULLS FIRST|LAST], ...] [LIMIT n [OFFSET m]]

  source := table [[AS] alias] [TABLESAMPLE BERNOULLI | SYSTEM (p) [REPEATABLE (seed)]] | ( select ) [AS] alias
  join   := [INNER | LEFT [OUTER] | RIGHT [OUTER] | FULL [OUTER] | CROSS] JOIN source [ON e]

Expressions: literals (incl. DATE '...', TIMESTAMP '...', INTERVAL '...' [unit]), [qualifier.]column,
+ - * / %, comparisons, AND OR NOT, IS [NOT] NULL, [NOT] BETWEEN, [NOT] IN (list), CAST(e AS type),
e [NOT] IN (select), [NOT] EXISTS (select), (select) as a scalar value,
e [NOT] LIKE | ILIKE 'pattern' [ESCAPE 'c'],
CASE WHEN, EXTRACT(field FROM e), FLOOR / CEIL(e TO unit), function calls incl. aggregates with
DISTINCT and FILTER (WHERE ...), and window calls  f(...) OVER ([PARTITION BY e, ...] [ORDER BY ...] [frame])
with frame := ROWS | RANGE  BETWEEN bound AND bound | bound,
     bound := UNBOUNDED PRECEDING | n PRECEDING | CURRENT ROW | n FOLLOWING | UNBOUNDED FOLLOWING.

Statements around the path (custom statements of the reference's parser, src/parser.rs):
  CREATE [OR REPLACE] TABLE|VIEW [IF NOT EXISTS] [schema.]name AS [(] query [)]
  CREATE [OR REPLACE] TABLE [IF NOT EXISTS] [schema.]name WITH (key = literal [, ...])
  DROP TABLE [IF EXISTS] [schema.]name
  ANALYZE TABLE [schema.]name COMPUTE STATISTICS FOR ALL COLUMNS | COLUMNS c1 [, c2 ...]
CREATE / DROP / TABLE / VIEW / IF / EXISTS / REPLACE / ANALYZE / COMPUTE / STATISTICS / FOR / COLUMNS and
TABLESAMPLE / BERNOULLI / SYSTEM / REPEATABLE, and OVER / PARTITION / ROWS / RANGE / UNBOUNDED / PRECEDING /
FOLLOWING / CURRENT / ROW are contextual words, not reserved.

Every RAND / RANDOM / RAND_INTEGER call and every TABLESAMPLE clause gets its call-site number `site`
(1, 2, 3 ... in textual order), which keys its random numbers apart from the statement's other ones.
"""
import re
from typing import List, Optional

from ..utils import ParsingException

_TOKEN = re.compile(r"""
    (?P<ws>\s+|--[^\n]*)
  | (?P<num>(?:\d+\.\d*|\.\d+|\d+)(?:[eE][+-]?\d+)?)
  | (?P<str>'(?:[^']|'')*')
  | (?P<qid>"(?:[^"]|"")*"|`[^`]*`)
  | (?P<id>[A-Za-z_][A-Za-z_0-9$]*)
  | (?P<op><>|!=|<=|>=|\|\||[-+*/%=<>(),.;])
""", re.X)

KEYWORDS = {"SELECT", "FROM", "WHERE", "GROUP", "BY", "HAVING", "ORDER", "LIMIT", "OFFSET", "AS", "AND", "OR",
            "NOT", "IS", "NULL", "IN", "BETWEEN", "JOIN", "INNER", "LEFT", "RIGHT", "FULL", "OUTER", "CROSS", "ON",
            "DISTINCT", "CASE", "WHEN", "THEN", "ELSE", "END", "CAST", "TRUE", "FALSE", "ASC", "DESC", "NULLS",
            "FIRST", "LAST", "WITH", "FILTER", "UNION", "ALL", "EXPLAIN", "SEMI", "ANTI", "USING"}


_LIKE_WORDS = ("LIKE", "ILIKE", "SIMILAR")
RAND_FUNCS = ("RAND", "RANDOM", "RAND_INTEGER")
_STRING_FUNCS = {"CONCAT", "UPPER", "LOWER", "SUBSTRING", "SUBSTR", "TRIM", "LTRIM", "RTRIM", "BTRIM", "POSITION",
                 "STRPOS", "CHAR_LENGTH", "CHARACTER_LENGTH", "LENGTH", "REPLACE", "INITCAP", "OVERLAY"}
_TIME_UNITS = {"YEAR", "QUARTER", "MONTH", "WEEK", "DAY", "HOUR", "MINUTE", "SECOND", "MILLISECOND", "MICROSECOND",
               "NANOSECOND"}


class Tok:
    __slots__ = ("kind", "val", "pos")

    def __init__(self, kind, val, pos):
        self.kind, self.val, self.pos = kind, val, pos

    def __repr__(self):
        return f"{self.kind}:{self.val}"


def tokenize(sql: str) -> List[Tok]:
    out, pos = [], 0
    while pos < len(sql):
        m = _TOKEN.match(sql, pos)
        if not m:
            raise ParsingException(sql, f"Unexpected character {sql[pos]!r} at position {pos}")
        pos = m.end()
        if m.lastgroup == "ws":
            continue
        v = m.group(m.lastgroup)
        if m.lastgroup == "id":
            up = v.upper()
            out.append(Tok("kw", up, m.start()) if up in KEYWORDS else Tok("id", v, m.start()))
        elif m.lastgroup == "qid":
            out.append(Tok("id", v[1:-1].replace('""', '"'), m.start()))
        elif m.lastgroup == "str":
            out.append(Tok("str", v[1:-1].replace("''", "'"), m.start()))
        else:
            out.append(Tok(m.lastgroup, v, m.start()))
    out.append(Tok("eof", "", len(sql)))
    return out


class Node(dict):
    """Syntax-tree node: a dict with attribute access."""
    __getattr__ = dict.get

    def __init__(self, kind, **kw):
        super().__init__(kind=kind, **kw)


class Parser:
    def __init__(self, sql: str):
        self.sql = sql
        self.toks = tokenize(sql)
        self.i = 0
        self.sites = 0           # call sites of RAND / TABLESAMPLE numbered so far

    # -- helpers
    @property
    def cur(self) -> Tok:
        return self.toks[self.i]

    def error(self, msg):
        raise ParsingException(self.sql, f"{msg} near position {self.cur.pos}: ...{self.sql[self.cur.pos:self.cur.pos + 30]!r}")

    def at_kw(self, *kws):
        return self.cur.kind == "kw" and self.cur.val in kws

    def at_op(self, *ops):
        return self.cur.kind == "op" and self.cur.val in ops

    def eat_kw(self, *kws):
        if self.at_kw(*kws):
            self.i += 1
            return self.toks[self.i - 1].val
        return None

    def eat_op(self, *ops):
        if self.at_op(*ops):
            self.i += 1
            return self.toks[self.i - 1].val
        return None

    def expect_kw(self, kw):
        if not self.eat_kw(kw):
            self.error(f"Expected {kw}")

    def expect_op(self, op):
        if not self.eat_op(op):
            self.error(f"Expected '{op}'")

    def ident(self):
        if self.cur.kind == "id":
            self.i += 1
            return self.toks[self.i - 1].val
        # non-reserved use of some keywords as identifiers (e.g. a column called "first")
        if self.cur.kind == "kw" and self.cur.val in ("FIRST", "LAST", "FILTER", "ALL"):
            self.i += 1
            return self.toks[self.i - 1].val.lower()
        self.error("Expected identifier")

    def at_word(self, *words):
        return self.cur.kind == "id" and self.cur.val.upper() in words

    def eat_word(self, *words):
        if self.at_word(*words):
            self.i += 1
            return self.toks[self.i - 1].val.upper()
        return None

    def expect_word(self, word):
        if not self.eat_word(word):
            self.error(f"Expected {word}")

    def qualified_name(self) -> str:
        parts = [self.ident()]
        while self.eat_op("."):
            parts.append(self.ident())
        return ".".join(parts)

    # -- statements
    def parse_ddl(self) -> Optional[Node]:
        if self.at_word("ANALYZE") and self.toks[self.i + 1].kind == "id":
            self.i += 1
            self.expect_word("TABLE")
            name = self.qualified_name()
            self.expect_word("COMPUTE")
            self.expect_word("STATISTICS")
            self.expect_word("FOR")
            columns = []
            if self.eat_kw("ALL"):
                self.expect_word("COLUMNS")
            else:
                self.expect_word("COLUMNS")
                columns.append(self.ident())
                while self.eat_op(","):
                    columns.append(self.ident())
            return Node("analyze_table", name=name, columns=columns)
        if self.at_word("DROP") and self.toks[self.i + 1].kind == "id":
            self.i += 1
            self.expect_word("TABLE")
            if_exists = False
            if self.at_word("IF"):
                self.i += 1
                self.expect_word("EXISTS")
                if_exists = True
            return Node("drop_table", name=self.qualified_name(), if_exists=if_exists)
        if not (self.at_word("CREATE") and self.toks[self.i + 1].kind in ("id", "kw")):
            return None
        self.i += 1
        or_replace = False
        if self.eat_kw("OR"):
            self.expect_word("REPLACE")
            or_replace = True
        what = self.eat_word("TABLE", "VIEW")
        if what is None:
            self.error("Expected TABLE or VIEW")
        if_not_exists = False
        if self.at_word("IF"):
            self.i += 1
            self.expect_kw("NOT")
            self.expect_word("EXISTS")
            if_not_exists = True
        name = self.qualified_name()
        if self.eat_kw("AS"):
            paren = bool(self.at_op("(") and self.toks[self.i + 1].kind == "kw"
                         and self.toks[self.i + 1].val in ("SELECT", "WITH") and self.eat_op("("))
            q = self.parse_query()
            if paren:
                self.expect_op(")")
            return Node("create_memory_table", name=name, query=q, or_replace=or_replace,
                        if_not_exists=if_not_exists, is_table=(what == "TABLE"))
        if what == "TABLE" and self.eat_kw("WITH"):
            self.expect_op("(")
            kwargs = {}
            while True:
                key = self.ident()
                self.expect_op("=")
                lit = self.parse_primary()
                neg = False
                if lit.kind != "lit":
                    self.error("Expected a literal value")
                kwargs[key] = lit.value
                if not self.eat_op(","):
                    break
            self.expect_op(")")
            return Node("create_table", name=name, kwargs=kwargs, or_replace=or_replace, if_not_exists=if_not_exists)
        self.error("Expected AS or WITH")

    def parse_statement(self) -> Node:
        ddl = self.parse_ddl()
        if ddl is not None:
            self.eat_op(";")
            if self.cur.kind != "eof":
                self.error("Unexpected trailing input")
            return ddl
        explain = bool(self.eat_kw("EXPLAIN"))
        q = self.parse_query()
        self.eat_op(";")
        if self.cur.kind != "eof":
            self.error("Unexpected trailing input")
        if explain:
            return Node("explain", query=q)
        return q

    def parse_query(self) -> Node:
        ctes = []
        if self.eat_kw("WITH"):
            while True:
                name = self.ident()
                self.expect_kw("AS")
                self.expect_op("(")
                ctes.append((name, self.parse_query()))
                self.expect_op(")")
                if not self.eat_op(","):
                    break
        q = self.parse_select()
        q["ctes"] = ctes
        return q

    def parse_select(self) -> Node:
        self.expect_kw("SELECT")
        distinct = bool(self.eat_kw("DISTINCT"))
        self.eat_kw("ALL")
        items = [self.parse_select_item()]
        while self.eat_op(","):
            items.append(self.parse_select_item())
        source = None
        if self.eat_kw("FROM"):
            source = self.parse_from()
        where = self.parse_expr() if self.eat_kw("WHERE") else None
        group_by = []
        if self.eat_kw("GROUP"):
            self.expect_kw("BY")
            group_by.append(self.parse_expr())
            while self.eat_op(","):
                group_by.append(self.parse_expr())
        having = self.parse_expr() if self.eat_kw("HAVING") else None
        if self.at_window_clause():
            raise NotImplementedError("the WINDOW clause (named windows) is not supported; write the window "
                                      "specification inline in OVER (...)")
        order_by = self.parse_order_items() if self.eat_kw("ORDER") else []
        limit = offset = None
        if self.eat_kw("LIMIT"):
            limit = self.parse_expr()
        if self.eat_kw("OFFSET"):
            offset = self.parse_expr()
        return Node("select", distinct=distinct, items=items, source=source, where=where, group_by=group_by,
                    having=having, order_by=order_by, limit=limit, offset=offset, ctes=[])

    def parse_select_item(self):
        if self.eat_op("*"):
            return (Node("star", qualifier=None), None)
        # qualifier.*
        if self.cur.kind == "id" and self.toks[self.i + 1].kind == "op" and self.toks[self.i + 1].val == "." \
                and self.toks[self.i + 2].kind == "op" and self.toks[self.i + 2].val == "*":
            q = self.ident()
            self.i += 2
            return (Node("star", qualifier=q), None)
        e = self.parse_expr()
        alias = None
        if self.eat_kw("AS"):
            alias = self.ident()
        elif self.cur.kind == "id":
            alias = self.ident()
        return (e, alias)

    def parse_from(self) -> Node:
        left = self.parse_source()
        while True:
            if self.eat_op(","):
                right = self.parse_source()
                left = Node("join", left=left, right=right, how="CROSS", on=None)
                continue
            how = None
            if self.eat_kw("INNER"):
                how = "INNER"
            elif self.eat_kw("LEFT"):
                how = "LEFT"
                if self.eat_kw("SEMI"):
                    how = "LEFTSEMI"
                elif self.eat_kw("ANTI"):
                    how = "LEFTANTI"
                else:
                    self.eat_kw("OUTER")
            elif self.eat_kw("RIGHT"):
                how = "RIGHT"
                self.eat_kw("OUTER")
            elif self.eat_kw("FULL"):
                how = "FULL"
                self.eat_kw("OUTER")
            elif self.eat_kw("CROSS"):
                how = "CROSS"
            if how is None and not self.at_kw("JOIN"):
                return left
            self.expect_kw("JOIN")
            right = self.parse_source()
            on = None
            if self.eat_kw("ON"):
                on = self.parse_expr()
            elif self.eat_kw("USING"):
                self.expect_op("(")
                cols = [self.ident()]
                while self.eat_op(","):
                    cols.append(self.ident())
                self.expect_op(")")
                on = Node("using", cols=cols)
            left = Node("join", left=left, right=right, how=how or "INNER", on=on)

    def parse_source(self) -> Node:
        if self.eat_op("("):
            q = self.parse_query()
            self.expect_op(")")
            self.eat_kw("AS")
            alias = self.ident()
            return Node("subquery", query=q, alias=alias, sample=self.parse_tablesample())
        parts = [self.ident()]
        while self.eat_op("."):
            parts.append(self.ident())
        alias = None
        if self.eat_kw("AS"):
            alias = self.ident()
        elif self.cur.kind == "id" and not self.at_tablesample() and not self.at_window_clause():
            alias = self.ident()
        return Node("table", name=parts, alias=alias, sample=self.parse_tablesample())

    def at_window_clause(self):
        """WINDOW name AS (...)"""
        return self.at_word("WINDOW") and self.toks[self.i + 1].kind == "id" and self.toks[self.i + 2].val == "AS"

    def at_tablesample(self):
        if not self.at_word("TABLESAMPLE"):
            return False
        nxt = self.toks[self.i + 1]
        return nxt.kind == "id" and nxt.val.upper() in ("BERNOULLI", "SYSTEM")

    def parse_tablesample(self) -> Optional[Node]:
        """TABLESAMPLE BERNOULLI | SYSTEM (p) [REPEATABLE (seed)]; p and seed are checked by the binder"""
        if not self.at_tablesample():
            return None
        self.i += 1
        method = self.eat_word("BERNOULLI", "SYSTEM").lower()
        self.sites += 1
        site = self.sites
        self.expect_op("(")
        p = self.parse_expr()
        self.expect_op(")")
        seed = None
        if self.eat_word("REPEATABLE"):
            self.expect_op("(")
            seed = self.parse_expr()
            self.expect_op(")")
        return Node("tablesample", method=method, p=p, seed=seed, site=site)

    # -- window functions
    def parse_over(self, call: Node) -> Node:
        """call OVER ([PARTITION BY e, ...] [ORDER BY e [ASC|DESC] [NULLS FIRST|LAST], ...] [frame])"""
        self.expect_word("OVER")
        if not self.at_op("("):
            raise NotImplementedError("a named window (OVER name / the WINDOW clause) is not supported; write the "
                                      "window specification inline")
        self.i += 1
        partition = []
        if self.eat_word("PARTITION"):
            self.expect_kw("BY")
            partition.append(self.parse_expr())
            while self.eat_op(","):
                partition.append(self.parse_expr())
        order = self.parse_order_items() if self.eat_kw("ORDER") else []
        frame = None
        if self.at_word("ROWS", "RANGE", "GROUPS"):
            frame = self.parse_frame()
        self.expect_op(")")
        return Node("window", func=call, partition=partition, order=order, frame=frame)

    def parse_frame(self) -> Node:
        unit = self.eat_word("ROWS", "RANGE", "GROUPS")
        if unit == "GROUPS":
            raise NotImplementedError("GROUPS window frames are not supported; use ROWS or RANGE")
        if self.eat_kw("BETWEEN"):
            lo = self.parse_frame_bound()
            self.expect_kw("AND")
            hi = self.parse_frame_bound()
        else:
            lo, hi = self.parse_frame_bound(), ("current", 0)
        if self.at_word("EXCLUDE"):
            raise NotImplementedError("EXCLUDE in a window frame is not supported")
        return Node("frame", unit=unit, lo=lo, hi=hi)

    def parse_frame_bound(self):
        """-> (kind, n): ("unbounded", -1 | +1), ("current", 0), ("offset", -n | +n)"""
        if self.eat_word("UNBOUNDED"):
            which = self.eat_word("PRECEDING", "FOLLOWING")
            if which is None:
                self.error("Expected PRECEDING or FOLLOWING")
            return ("unbounded", -1 if which == "PRECEDING" else 1)
        if self.eat_word("CURRENT"):
            self.expect_word("ROW")
            return ("current", 0)
        if self.cur.kind != "num" or not re.fullmatch(r"\d+", self.cur.val):
            self.error("A window frame offset is a non-negative integer literal")
        k = int(self.cur.val)
        self.i += 1
        which = self.eat_word("PRECEDING", "FOLLOWING")
        if which is None:
            self.error("Expected PRECEDING or FOLLOWING")
        return ("offset", -k if which == "PRECEDING" else k)

    def parse_order_items(self):
        self.expect_kw("BY")
        out = []
        while True:
            e = self.parse_expr()
            asc = True
            if self.eat_kw("DESC"):
                asc = False
            else:
                self.eat_kw("ASC")
            nulls_first = None
            if self.eat_kw("NULLS"):
                nulls_first = bool(self.eat_kw("FIRST"))
                if not nulls_first:
                    self.expect_kw("LAST")
            out.append((e, asc, nulls_first))
            if not self.eat_op(","):
                return out

    # -- expressions (precedence climbing)
    def parse_expr(self) -> Node:
        return self.parse_or()

    def parse_or(self):
        e = self.parse_and()
        while self.eat_kw("OR"):
            e = Node("bin", op="OR", l=e, r=self.parse_and())
        return e

    def parse_and(self):
        e = self.parse_not()
        while self.eat_kw("AND"):
            e = Node("bin", op="AND", l=e, r=self.parse_not())
        return e

    def parse_not(self):
        if self.eat_kw("NOT"):
            return Node("not", e=self.parse_not())
        return self.parse_cmp()

    def parse_cmp(self):
        e = self.parse_add()
        while True:
            if self.at_op("=", "<>", "!=", "<", "<=", ">", ">="):
                op = self.eat_op("=", "<>", "!=", "<", "<=", ">", ">=")
                if (self.at_kw("ALL") or self.at_word("ANY", "SOME")) and self.toks[self.i + 1].val == "(":
                    raise NotImplementedError("ANY / ALL / SOME (subquery) comparisons are not supported; write "
                                              "[NOT] IN (SELECT ...) or [NOT] EXISTS (SELECT ...)")
                e = Node("bin", op="!=" if op == "<>" else op, l=e, r=self.parse_add())
            elif self.at_kw("IS"):
                self.i += 1
                neg = bool(self.eat_kw("NOT"))
                if self.eat_kw("NULL"):
                    e = Node("isnull", e=e, negated=neg)
                elif self.eat_kw("TRUE"):
                    e = Node("istrue", e=e, negated=neg, value=True)
                elif self.eat_kw("FALSE"):
                    e = Node("istrue", e=e, negated=neg, value=False)
                elif self.eat_word("UNKNOWN"):      # a boolean is UNKNOWN iff it is NULL (call.py:1123-1124)
                    e = Node("isnull", e=e, negated=neg)
                else:
                    self.error("Expected NULL, TRUE, FALSE or UNKNOWN after IS")
            elif self.at_kw("NOT") and self.toks[self.i + 1].kind == "kw" and self.toks[self.i + 1].val in ("BETWEEN", "IN"):
                self.i += 1
                e = self._between_or_in(e, True)
            elif self.at_kw("BETWEEN", "IN"):
                e = self._between_or_in(e, False)
            elif self.at_word(*_LIKE_WORDS) or (self.at_kw("NOT") and self.toks[self.i + 1].kind == "id"
                                                and self.toks[self.i + 1].val.upper() in _LIKE_WORDS):
                negated = bool(self.eat_kw("NOT"))
                e = self._like(e, negated)
            else:
                return e

    def _between_or_in(self, e, negated):
        if self.eat_kw("BETWEEN"):
            lo = self.parse_add()
            self.expect_kw("AND")
            hi = self.parse_add()
            return Node("between", e=e, lo=lo, hi=hi, negated=negated)
        self.expect_kw("IN")
        self.expect_op("(")
        if self.at_kw("SELECT", "WITH"):
            q = self.parse_query()
            self.expect_op(")")
            return Node("insubquery", e=e, query=q, negated=negated)
        items = [self.parse_expr()]
        while self.eat_op(","):
            items.append(self.parse_expr())
        self.expect_op(")")
        return Node("inlist", e=e, items=items, negated=negated)

    def _like(self, e, negated):
        word = self.eat_word(*_LIKE_WORDS)
        if word == "SIMILAR":
            raise NotImplementedError("SIMILAR TO is not supported; use LIKE / ILIKE")
        pattern = self.parse_add()
        escape = None
        if self.eat_word("ESCAPE"):
            if self.cur.kind != "str" or len(self.cur.val) != 1:
                self.error("ESCAPE takes a string of one character")
            escape = self.cur.val
            self.i += 1
        return Node("like", e=e, pattern=pattern, escape=escape, negated=negated, ilike=word == "ILIKE")

    def parse_add(self):
        e = self.parse_mul()
        if self.at_op("||"):
            raise NotImplementedError("string concatenation (||) is not supported: VARCHAR values are dictionary "
                                      "codes here")
        while self.at_op("+", "-"):
            op = self.eat_op("+", "-")
            e = Node("bin", op=op, l=e, r=self.parse_mul())
        return e

    def parse_mul(self):
        e = self.parse_unary()
        while self.at_op("*", "/", "%"):
            op = self.eat_op("*", "/", "%")
            e = Node("bin", op=op, l=e, r=self.parse_unary())
        return e

    def parse_unary(self):
        if self.eat_op("-"):
            inner = self.parse_unary()
            if inner.kind == "lit" and isinstance(inner.value, (int, float)) and not isinstance(inner.value, bool):
                return Node("lit", value=-inner.value)
            return Node("neg", e=inner)
        if self.eat_op("+"):
            return self.parse_unary()
        return self.parse_primary()

    def parse_primary(self):
        t = self.cur
        if t.kind == "num":
            self.i += 1
            txt = t.val
            if re.fullmatch(r"\d+", txt):
                return Node("lit", value=int(txt))
            return Node("lit", value=float(txt))
        if t.kind == "str":
            self.i += 1
            return Node("lit", value=t.val)
        if self.eat_kw("TRUE"):
            return Node("lit", value=True)
        if self.eat_kw("FALSE"):
            return Node("lit", value=False)
        if self.eat_kw("NULL"):
            return Node("lit", value=None)
        if self.eat_op("("):
            if self.at_kw("SELECT", "WITH"):                # (SELECT one_value ...) as an expression
                q = self.parse_query()
                self.expect_op(")")
                return Node("scalarsubquery", query=q)
            e = self.parse_expr()
            if self.at_op(","):
                raise NotImplementedError("row values such as (a, b) IN (SELECT ...) are not supported; compare "
                                          "one expression, or write a correlated EXISTS")
            self.expect_op(")")
            return e
        if self.at_word("EXISTS") and self.toks[self.i + 1].val == "(" and self.toks[self.i + 2].kind == "kw" \
                and self.toks[self.i + 2].val in ("SELECT", "WITH"):
            self.i += 2
            q = self.parse_query()
            self.expect_op(")")
            return Node("exists", query=q)
        if self.eat_kw("CAST"):
            self.expect_op("(")
            e = self.parse_expr()
            self.expect_kw("AS")
            ty = self.ident()
            if ty.upper() == "DOUBLE" and self.cur.kind == "id" and self.cur.val.upper() == "PRECISION":
                self.i += 1
            if self.eat_op("("):  # DECIMAL(p, s) and friends
                while not self.eat_op(")"):
                    self.i += 1
            self.expect_op(")")
            return Node("cast", e=e, type=ty.upper())
        if self.eat_kw("CASE"):
            operand = None
            if not self.at_kw("WHEN"):
                operand = self.parse_expr()
            whens = []
            while self.eat_kw("WHEN"):
                w = self.parse_expr()
                self.expect_kw("THEN")
                whens.append((Node("bin", op="=", l=operand, r=w) if operand is not None else w, self.parse_expr()))
            other = self.parse_expr() if self.eat_kw("ELSE") else None
            self.expect_kw("END")
            return Node("case", whens=whens, other=other)
        nxt = self.toks[self.i + 1] if self.i + 1 < len(self.toks) else t
        if t.kind == "id" and t.val.upper() in ("DATE", "TIMESTAMP") and nxt.kind == "str":
            self.i += 2                                   # DATE 'YYYY-MM-DD', TIMESTAMP 'YYYY-MM-DD HH:MM:SS'
            return Node("typed_lit", type=t.val.upper(), value=nxt.val)
        if t.kind == "id" and t.val.upper() == "INTERVAL" and nxt.kind == "str":
            self.i += 2                                   # INTERVAL '4 days' | INTERVAL '4' DAY
            unit = self.ident().upper() if self.cur.kind == "id" and self.cur.val.upper().rstrip("S") in _TIME_UNITS \
                else None
            return Node("interval", value=nxt.val, unit=unit)
        if t.kind == "id" and t.val.upper() in _STRING_FUNCS and nxt.kind == "op" and nxt.val == "(":
            raise NotImplementedError(f"{t.val.upper()}: string functions are not supported; VARCHAR columns are "
                                      "compared, matched with [NOT] LIKE / ILIKE, grouped, sorted and joined on")
        if t.kind == "id" and t.val.upper() == "EXTRACT" and nxt.kind == "op" and nxt.val == "(":
            self.i += 2                                   # EXTRACT(field FROM x)
            field = self.ident().upper()
            self.expect_kw("FROM")
            x = self.parse_expr()
            self.expect_op(")")
            return Node("func", name="EXTRACT", args=[Node("lit", value=field), x], distinct=False, star=False,
                        filter=None)
        if t.kind == "id" or (t.kind == "kw" and t.val in ("LEFT", "RIGHT", "FIRST", "LAST", "FILTER")
                              and self.toks[self.i + 1].kind == "op" and self.toks[self.i + 1].val in ("(", ".")):
            name = self.ident() if t.kind == "id" else (self.toks[self.i].val, setattr(self, "i", self.i + 1))[0]
            if name.upper() in RAND_FUNCS and self.at_op("("):
                self.sites += 1
                site = self.sites
                self.i += 1
                args = []
                if not self.at_op(")"):
                    args.append(self.parse_expr())
                    while self.eat_op(","):
                        args.append(self.parse_expr())
                self.expect_op(")")
                return Node("func", name=name.upper(), args=args, distinct=False, star=False, filter=None, site=site)
            if self.eat_op("("):  # function call
                distinct = bool(self.eat_kw("DISTINCT"))
                args, star = [], False
                if self.eat_op("*"):
                    star = True
                elif not self.at_op(")"):
                    args.append(self.parse_expr())
                    if name.upper() in ("FLOOR", "CEIL") and self.eat_word("TO"):   # FLOOR(x TO unit)
                        args.append(Node("lit", value=self.ident().upper()))
                        self.expect_op(")")
                        return Node("func", name="TIMESTAMP" + name.upper(), args=args, distinct=False,
                                    star=False, filter=None)
                    while self.eat_op(","):
                        args.append(self.parse_expr())
                self.expect_op(")")
                filt = None
                if self.at_kw("FILTER") and self.toks[self.i + 1].kind == "op" and self.toks[self.i + 1].val == "(":
                    self.i += 2
                    self.expect_kw("WHERE")
                    filt = self.parse_expr()
                    self.expect_op(")")
                call = Node("func", name=name.upper(), args=args, distinct=distinct, star=star, filter=filt)
                if self.at_word("OVER"):
                    return self.parse_over(call)
                return call
            parts = [name]
            while self.eat_op("."):
                parts.append(self.ident())
            return Node("col", parts=parts)
        self.error("Unexpected token")


def parse_sql(sql: str) -> Node:
    return Parser(sql).parse_statement()
