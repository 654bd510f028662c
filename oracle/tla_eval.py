"""tla_eval.py — TEST INFRASTRUCTURE (like everything under oracle/): a small evaluator for the TLA+ subset that
vsr-revisited/paper/VSR.tla of the reference is written in.

Why: the C++ oracle (vsr_oracle.cpp) is my restatement of the spec; TLC — the tool that gives the spec its meaning — is
not in this image (no JVM).  This module executes the reference's OWN SOURCE TEXT: it parses VSR.tla as it lies under
the reference (Vanlightly/vsr-tlaplus) and enumerates Init and the successors of a state the way TLC does (conjuncts left to right, x' = e
assigns the first time and tests afterwards, \\E and \\/ branch, UNCHANGED copies, operator definitions are expanded).
tests/test_spec_text.py compares, state by state, the successor sets it derives from the text with the oracle's, and
whole small state spaces level by level.  It pins the oracle to the spec's text rather than to my reading of it.

Scope: exactly the constructs VSR.tla uses (junction lists by column, \\E/\\A/CHOOSE, LET, IF, records, functions, EXCEPT
with @ and nested paths, sets, sequences, Quantify/LAMBDA, Permutations, model values).  Not a general TLA+ tool, no
liveness, no TLC value ORDER: CHOOSE takes the first candidate in this module's own order and REPORTS when more than one
candidate satisfied the predicate (see Evaluator.choose_log), so a caller can tell whether a result depended on the pick.
Nothing here is imported by the product; the tests replay what it answered on the spec's text (tests/spec_text.py).
"""
import re
from itertools import permutations, product

# ------------------------------------------------------------------------------------------------ values


class ModelValue:
    __slots__ = ("name",)
    _pool = {}

    def __new__(cls, name):
        v = cls._pool.get(name)
        if v is None:
            v = object.__new__(cls)
            v.name = name
            cls._pool[name] = v
        return v

    def __repr__(self):
        return self.name


class Fn:
    """a TLA+ function with a finite domain: records (string keys), sequences/tuples (keys 1..n), bags, ..."""
    __slots__ = ("d", "_h", "_k")

    def __init__(self, d):
        self.d = d
        self._h = None
        self._k = None

    def __hash__(self):
        if self._h is None:
            self._h = hash(frozenset(self.d.items()))
        return self._h

    def __eq__(self, o):
        return isinstance(o, Fn) and self.d == o.d

    def __ne__(self, o):
        return not self.__eq__(o)

    def is_seq(self):
        n = len(self.d)
        return all(isinstance(k, int) and not isinstance(k, bool) for k in self.d) and set(self.d) == set(range(1, n + 1))

    def __repr__(self):
        return fmt(self)


EMPTY = Fn({})


def seq(items):
    return Fn({i + 1: v for i, v in enumerate(items)})


class EvalError(Exception):
    pass


def vkey(v):
    """a total order on values (this module's own; NOT TLC's)"""
    if isinstance(v, bool):
        return (0, int(v))
    if isinstance(v, int):
        return (1, v)
    if isinstance(v, str):
        return (2, v)
    if isinstance(v, ModelValue):
        return (3, v.name)
    if isinstance(v, frozenset):
        return (4, len(v), tuple(sorted(vkey(x) for x in v)))
    if isinstance(v, Fn):
        if v._k is None:
            v._k = (5, len(v.d), tuple(sorted((vkey(k), vkey(x)) for k, x in v.d.items())))
        return v._k
    raise EvalError("no order for %r" % (v,))


def ordered(s):
    return sorted(s, key=vkey)


def fmt(v):
    """TLC-style text of a value"""
    if isinstance(v, bool):
        return "TRUE" if v else "FALSE"
    if isinstance(v, int):
        return str(v)
    if isinstance(v, str):
        return '"%s"' % v
    if isinstance(v, ModelValue):
        return v.name
    if isinstance(v, frozenset):
        if v and all(isinstance(x, int) and not isinstance(x, bool) for x in v) and set(v) == set(range(min(v), max(v) + 1)):
            return "%d..%d" % (min(v), max(v))
        return "{" + ", ".join(fmt(x) for x in ordered(v)) + "}"
    if isinstance(v, Fn):
        if not v.d:
            return "<<>>"
        if v.is_seq():
            return "<<" + ", ".join(fmt(v.d[i]) for i in range(1, len(v.d) + 1)) + ">>"
        if all(isinstance(k, str) for k in v.d):
            return "[" + ", ".join("%s |-> %s" % (k, fmt(x)) for k, x in v.d.items()) + "]"
        return "(" + " @@ ".join("%s :> %s" % (fmt(k), fmt(v.d[k])) for k in ordered(v.d)) + ")"
    raise EvalError("cannot print %r" % (v,))


# ------------------------------------------------------------------------------------------------ tokens

TOKEN_RE = re.compile(r"""
    (?P<ws>[ \t\r]+) | (?P<nl>\n) |
    (?P<num>\d+) |
    (?P<str>"[^"\n]*") |
    (?P<id>[A-Za-z_][A-Za-z0-9_]*) |
    (?P<op>/\\|\\/|\\[A-Za-z]+|\\|==|=>|=<|\|->|->|<<|>>|<=>|<=|>=|/=|\.\.|:>|@@|[=<>.:@\#'!~+\-*%()\[\]{},|])
""", re.X)

KEYWORDS = {"IF", "THEN", "ELSE", "LET", "IN", "CHOOSE", "EXCEPT", "UNCHANGED", "DOMAIN", "LAMBDA", "SUBSET", "UNION", "ENABLED",
            "TRUE", "FALSE", "CONSTANT", "CONSTANTS", "VARIABLE", "VARIABLES", "EXTENDS", "MODULE", "ASSUME", "THEOREM", "LOCAL", "INSTANCE"}


class Tok:
    __slots__ = ("kind", "text", "line", "col")

    def __init__(self, kind, text, line, col):
        self.kind, self.text, self.line, self.col = kind, text, line, col

    def __repr__(self):
        return "%s:%r@%d:%d" % (self.kind, self.text, self.line, self.col)


def strip_comments(text):
    out, i, depth, n = [], 0, 0, len(text)
    while i < n:
        if text.startswith("(*", i):
            depth += 1
            out.append("  ")
            i += 2
        elif depth and text.startswith("*)", i):
            depth -= 1
            out.append("  ")
            i += 2
        elif depth:
            out.append("\n" if text[i] == "\n" else " ")
            i += 1
        elif text.startswith("\\*", i):
            j = text.find("\n", i)
            j = n if j < 0 else j
            out.append(" " * (j - i))
            i = j
        else:
            out.append(text[i])
            i += 1
    return "".join(out)


def tokenize(text):
    text = strip_comments(text)
    text = "\n".join("" if re.match(r"^\s*(-{4,}.*|={4,}\s*)$", ln) else ln for ln in text.split("\n"))
    toks, line, linestart, i = [], 1, 0, 0
    while i < len(text):
        m = TOKEN_RE.match(text, i)
        if not m:
            raise EvalError("cannot tokenize at line %d: %r" % (line, text[i:i + 20]))
        kind = m.lastgroup
        if kind == "nl":
            line += 1
            linestart = m.end()
        elif kind != "ws":
            t = m.group()
            if kind == "id" and t in KEYWORDS:
                kind = "kw"
            toks.append(Tok(kind, t, line, m.start() - linestart))
        i = m.end()
    toks.append(Tok("eof", "", line + 1, -1))
    return toks


# ------------------------------------------------------------------------------------------------ parser

BINOPS = {"=>": 1, "<=>": 2, "/\\": 3, "\\/": 3, "=": 5, "#": 5, "/=": 5, "<": 5, ">": 5, "<=": 5, "=<": 5, ">=": 5, "\\in": 5,
          "\\notin": 5, "\\subseteq": 5, "@@": 6, ":>": 7, "\\": 8, "\\union": 8, "\\cup": 8, "\\cap": 8, "\\intersect": 8, "..": 9,
          "+": 10, "-": 10, "%": 11, "*": 13, "\\div": 13, "\\o": 13}


class Parser:
    def __init__(self, toks):
        self.t, self.p, self.j = toks, 0, []

    def peek(self, k=0):
        return self.t[min(self.p + k, len(self.t) - 1)]

    def next(self):
        tok = self.t[self.p]
        self.p += 1
        return tok

    def expect(self, text):
        tok = self.next()
        if tok.text != text:
            raise EvalError("expected %r, found %r" % (text, tok))
        return tok

    def blocked(self):
        """a token at or left of the innermost junction list's bullet column ends the current item"""
        tok = self.peek()
        return tok.kind == "eof" or (self.j and tok.col <= self.j[-1])

    def delim(self, fn):
        self.j.append(-1)  # the column rule is suspended inside brackets
        try:
            return fn()
        finally:
            self.j.pop()

    def expr(self, minp=0):
        left = self.prefix()
        while not self.blocked():
            tok = self.peek()
            if tok.kind == "op" and tok.text in BINOPS and BINOPS[tok.text] >= minp:
                self.next()
                right = self.expr(BINOPS[tok.text] + 1)
                left = ("bin", tok.text, left, right)
            else:
                break
        return left

    def postfix(self, e):
        while not self.blocked():
            tok = self.peek()
            if tok.text == "[" and tok.kind == "op":
                self.next()
                args = self.delim(lambda: self.exprlist("]"))
                e = ("app", e, args[0] if len(args) == 1 else ("tuple", args))
            elif tok.text == "." and tok.kind == "op" and self.peek(1).kind == "id":
                self.next()
                e = ("dot", e, self.next().text)
            elif tok.text == "'" and tok.kind == "op":
                self.next()
                e = ("prime", e)
            else:
                break
        return e

    def exprlist(self, close):
        items = []
        if self.peek().text == close:
            self.next()
            return items
        while True:
            items.append(self.expr(0))
            tok = self.next()
            if tok.text == close:
                return items
            if tok.text != ",":
                raise EvalError("expected ',' or %r, found %r" % (close, tok))

    def bounds(self):
        """x \\in S, y, z \\in T   ->  [([x], S), ([y, z], T)]"""
        groups = []
        while True:
            names = [self.next().text]
            while self.peek().text == ",":
                self.next()
                names.append(self.next().text)
            self.expect("\\in")
            groups.append((names, self.expr(6)))
            if self.peek().text == ",":
                self.next()
                continue
            return groups

    def prefix(self):
        tok = self.peek()
        k, t = tok.kind, tok.text
        if k == "op" and t in ("/\\", "\\/"):
            col, items = tok.col, []
            while self.peek().kind == "op" and self.peek().text == t and self.peek().col == col:
                self.next()
                self.j.append(col)
                try:
                    items.append(self.expr(0))
                finally:
                    self.j.pop()
            return ("and" if t == "/\\" else "or", items)
        self.next()
        if k == "num":
            return self.postfix(("lit", int(t)))
        if k == "str":
            return self.postfix(("lit", t[1:-1]))
        if k == "kw":
            if t in ("TRUE", "FALSE"):
                return ("lit", t == "TRUE")
            if t == "IF":
                c = self.expr(0)
                self.expect("THEN")
                a = self.expr(0)
                self.expect("ELSE")
                return ("if", c, a, self.expr(0))
            if t == "LET":
                defs = []
                while self.peek().text != "IN":
                    name = self.next().text
                    params = []
                    if self.peek().text == "(":
                        self.next()
                        while True:
                            params.append(self.next().text)
                            if self.next().text == ")":
                                break
                    self.expect("==")
                    defs.append((name, params, self.expr(0)))
                self.expect("IN")
                return ("let", defs, self.expr(0))
            if t == "CHOOSE":
                name = self.next().text
                self.expect("\\in")
                s = self.expr(6)
                self.expect(":")
                return ("choose", name, s, self.expr(0))
            if t == "UNCHANGED":
                return ("unchanged", self.expr(4))
            if t == "DOMAIN":
                return ("domain", self.expr(9))
            if t == "SUBSET":
                return ("subset", self.expr(8))
            if t == "UNION":
                return ("bigunion", self.expr(8))
            if t == "LAMBDA":
                params = [self.next().text]
                while self.peek().text == ",":
                    self.next()
                    params.append(self.next().text)
                self.expect(":")
                return ("lambda", params, self.expr(0))
            raise EvalError("unexpected keyword %r" % tok)
        if k == "id":
            if self.peek().text == "(" and self.peek().line == tok.line and self.peek().col == tok.col + len(t):
                self.next()
                args = self.delim(lambda: self.exprlist(")"))
                return self.postfix(("call", t, args))
            return self.postfix(("id", t))
        if t in ("\\E", "\\A"):
            groups = self.bounds()
            self.expect(":")
            return ("exists" if t == "\\E" else "forall", groups, self.expr(0))
        if t == "~":
            return ("not", self.expr(4))
        if t == "-":
            return ("neg", self.expr(12))
        if t == "(":
            e = self.delim(lambda: self.expr(0))
            self.expect(")")
            return self.postfix(e)
        if t == "<<":
            return self.postfix(("tuple", self.delim(lambda: self.exprlist(">>"))))
        if t == "{":
            return self.postfix(self.delim(self.setexpr))
        if t == "[":
            return self.postfix(self.delim(self.bracket))
        if t == "@":
            return self.postfix(("at",))
        raise EvalError("unexpected token %r" % tok)

    def setexpr(self):
        if self.peek().text == "}":
            self.next()
            return ("setenum", [])
        first = self.expr(0)
        tok = self.next()
        if tok.text == ":":
            if first[0] == "bin" and first[1] == "\\in" and first[2][0] == "id":  # {x \in S : P}
                pred = self.expr(0)
                self.expect("}")
                return ("setfilter", first[2][1], first[3], pred)
            groups = self.bounds()                                                 # {e : x \in S}
            self.expect("}")
            return ("setmap", first, groups)
        items = [first]
        while tok.text == ",":
            items.append(self.expr(0))
            tok = self.next()
        if tok.text != "}":
            raise EvalError("expected '}', found %r" % tok)
        return ("setenum", items)

    def bracket(self):
        a, b = self.peek(), self.peek(1)
        if a.kind == "id" and b.text == "|->":                                     # record
            fields = []
            while True:
                name = self.next().text
                self.expect("|->")
                fields.append((name, self.expr(0)))
                tok = self.next()
                if tok.text == "]":
                    return ("record", fields)
                if tok.text != ",":
                    raise EvalError("record: %r" % tok)
        if a.kind == "id" and b.text == ":":                                        # record SET (types; never evaluated)
            depth = 1
            while depth:
                tok = self.next()
                depth += tok.text == "["
                depth -= tok.text == "]"
            return ("typeexpr",)
        if a.kind == "id" and b.text in ("\\in", ","):                              # function constructor
            groups = self.bounds()
            self.expect("|->")
            body = self.expr(0)
            self.expect("]")
            return ("fcons", groups, body)
        e = self.expr(0)
        tok = self.next()
        if tok.text == "EXCEPT":
            specs = []
            while True:
                self.expect("!")
                path = []
                while self.peek().text in ("[", "."):
                    if self.next().text == "[":
                        args = self.exprlist("]")
                        path.append(("idx", args[0] if len(args) == 1 else ("tuple", args)))
                    else:
                        path.append(("fld", self.next().text))
                self.expect("=")
                specs.append((path, self.expr(0)))
                tok = self.next()
                if tok.text == "]":
                    return ("except", e, specs)
                if tok.text != ",":
                    raise EvalError("EXCEPT: %r" % tok)
        if tok.text in ("->", "|->"):                                               # function SET (types; never evaluated)
            depth = 1
            while depth:
                tok = self.next()
                depth += tok.text == "["
                depth -= tok.text == "]"
            return ("typeexpr",)
        raise EvalError("bracket expression: %r" % tok)


def parse_expression(text):
    p = Parser(tokenize(text))
    e = p.expr(0)
    if p.peek().kind != "eof":
        raise EvalError("trailing input at %r" % p.peek())
    return e


class Module:
    """top-level definitions of a module, parsed on first use (type definitions are never needed)"""

    def __init__(self, text):
        self.toks = tokenize(text)
        self.variables, self.constants, self.defs, self._parsed = [], [], {}, {}
        t, i, n = self.toks, 0, len(self.toks)
        starts = []
        while i < n - 1:
            tok = t[i]
            if tok.col == 0 and tok.kind == "kw" and tok.text in ("CONSTANT", "CONSTANTS", "VARIABLE", "VARIABLES", "EXTENDS"):
                j = i + 1
                names = []
                while t[j].kind == "id" or t[j].text == ",":
                    if t[j].kind == "id" and t[j].col != 0:
                        names.append(t[j].text)
                    elif t[j].kind == "id" and t[j].col == 0:
                        break
                    j += 1
                if tok.text.startswith("CONSTANT"):
                    self.constants += names
                elif tok.text.startswith("VARIABLE"):
                    self.variables += names
                i = j
                continue
            if tok.col == 0 and tok.kind == "id":
                j, params = i + 1, []
                if t[j].text == "(":
                    j += 1
                    while t[j].text != ")":
                        if t[j].kind == "id":
                            params.append(t[j].text)
                        j += 1
                    j += 1
                if t[j].text == "==":
                    starts.append((tok.text, params, j + 1, i))
            i += 1
        for k, (name, params, body_start, head) in enumerate(starts):
            end = starts[k + 1][3] if k + 1 < len(starts) else n - 1
            # a CONSTANTS/VARIABLES/... block between two definitions also ends the body
            for m in range(body_start, end):
                if self.toks[m].col == 0 and self.toks[m].kind == "kw":
                    end = m
                    break
            self.defs[name] = (params, body_start, end)

    def body(self, name):
        if name not in self._parsed:
            params, a, b = self.defs[name]
            toks = self.toks[a:b] + [Tok("eof", "", 0, -1)]
            p = Parser(toks)
            e = p.expr(0)
            if p.peek().kind != "eof":
                raise EvalError("definition %s: trailing input at %r" % (name, p.peek()))
            self._parsed[name] = (params, e)
        return self._parsed[name]


# ------------------------------------------------------------------------------------------------ evaluator


class Closure:
    __slots__ = ("params", "body", "env")

    def __init__(self, params, body, env):
        self.params, self.body, self.env = params, body, env


class Evaluator:
    def __init__(self, module, constants):
        self.m = module
        self.c = dict(constants)
        self.varset = set(module.variables)
        self.s = None          # current state: dict variable -> value
        self.sp = None         # next state being built (dict), None outside of action evaluation
        self.choose_log = []   # (number of candidates,) for every CHOOSE with more than one candidate since last cleared
        self.choose_pick = 0   # which candidate an ambiguous CHOOSE takes (tests retry with others)
        self._primed = {}

    # ---- names
    def lookup(self, name, env):
        if name in env:
            v = env[name]
            if isinstance(v, Closure) and not v.params:
                return self.ev(v.body, v.env)
            return v
        if name in self.c:
            return self.c[name]
        if name in self.varset:
            return self.s[name]
        if name in self.m.defs:
            params, body = self.m.body(name)
            if params:
                return Closure(params, body, {})
            return self.ev(body, {})
        if name == "Nat":
            raise EvalError("Nat is not enumerable")
        raise EvalError("unknown identifier %s" % name)

    def call(self, name, args, env):
        f = BUILTINS.get(name)
        if name in env or name in self.m.defs:
            if name in env:
                clo = env[name]
            else:
                params, body = self.m.body(name)
                clo = Closure(params, body, {})
            e2 = dict(clo.env)
            e2.update(zip(clo.params, args))
            return self.ev(clo.body, e2)
        if f:
            return f(self, *args)
        raise EvalError("unknown operator %s" % name)

    def apply_closure(self, clo, vals):
        e2 = dict(clo.env)
        e2.update(zip(clo.params, vals))
        return self.ev(clo.body, e2)

    def bindings(self, groups, env):
        """all assignments of the bound names of \\E / \\A / function constructors, in this module's set order"""
        doms = []
        names = []
        for ns, sexpr in groups:
            s = self.ev(sexpr, env)
            if not isinstance(s, frozenset):
                raise EvalError("quantifier domain is not a set: %s" % fmt(s))
            for nme in ns:
                names.append(nme)
                doms.append(ordered(s))
        for combo in product(*doms):
            e2 = dict(env)
            e2.update(zip(names, combo))
            yield e2, combo

    # ---- expressions
    def ev(self, n, env):
        k = n[0]
        if k == "lit":
            return n[1]
        if k == "id":
            return self.lookup(n[1], env)
        if k == "prime":
            if n[1][0] != "id" or n[1][1] not in self.varset:
                raise EvalError("prime of a non-variable")
            if self.sp is None or n[1][1] not in self.sp:
                raise EvalError("%s' read before it is determined" % n[1][1])
            return self.sp[n[1][1]]
        if k == "bin":
            return self.binop(n[1], n[2], n[3], env)
        if k == "and":
            for it in n[1]:
                if self.ev(it, env) is not True:
                    return False
            return True
        if k == "or":
            for it in n[1]:
                if self.ev(it, env) is True:
                    return True
            return False
        if k == "not":
            return not self.truth(self.ev(n[1], env))
        if k == "neg":
            return -self.ev(n[1], env)
        if k == "if":
            return self.ev(n[2], env) if self.truth(self.ev(n[1], env)) else self.ev(n[3], env)
        if k == "let":
            e2 = dict(env)
            for name, params, body in n[1]:
                e2[name] = Closure(params, body, e2)  # later definitions see earlier ones (and themselves: harmless)
            return self.ev(n[2], e2)
        if k == "call":
            args = [self.ev(a, env) if a[0] != "lambda" else Closure(a[1], a[2], env) for a in n[2]]
            return self.call(n[1], args, env)
        if k == "lambda":
            return Closure(n[1], n[2], env)
        if k == "app":
            f = self.ev(n[1], env)
            x = self.ev(n[2], env)
            if not isinstance(f, Fn):
                raise EvalError("applying a non-function %s" % fmt(f))
            if x not in f.d:
                raise EvalError("%s is not in the domain of %s" % (fmt(x), fmt(f)))
            return f.d[x]
        if k == "dot":
            r = self.ev(n[1], env)
            if not isinstance(r, Fn) or n[2] not in r.d:
                raise EvalError("record %s has no field %s" % (fmt(r) if isinstance(r, (Fn, frozenset, int)) else r, n[2]))
            return r.d[n[2]]
        if k == "tuple":
            return seq([self.ev(x, env) for x in n[1]])
        if k == "record":
            return Fn({name: self.ev(e, env) for name, e in n[1]})
        if k == "setenum":
            return frozenset(self.ev(x, env) for x in n[1])
        if k == "setfilter":
            s = self.ev(n[2], env)
            out = []
            for x in ordered(s):
                e2 = dict(env)
                e2[n[1]] = x
                if self.truth(self.ev(n[3], e2)):
                    out.append(x)
            return frozenset(out)
        if k == "setmap":
            return frozenset(self.ev(n[1], e2) for e2, _ in self.bindings(n[2], env))
        if k == "fcons":
            d = {}
            for e2, combo in self.bindings(n[1], env):
                d[combo[0] if len(combo) == 1 else seq(combo)] = self.ev(n[2], e2)
            return Fn(d)
        if k == "except":
            f = self.ev(n[1], env)
            for path, rhs in n[2]:
                f = self.except_one(f, path, rhs, env)
            return f
        if k == "at":
            return env["@"]
        if k == "domain":
            f = self.ev(n[1], env)
            if not isinstance(f, Fn):
                raise EvalError("DOMAIN of a non-function")
            return frozenset(f.d)
        if k == "exists":
            return any(self.truth(self.ev(n[2], e2)) for e2, _ in self.bindings(n[1], env))
        if k == "forall":
            return all(self.truth(self.ev(n[2], e2)) for e2, _ in self.bindings(n[1], env))
        if k == "choose":
            s = self.ev(n[2], env)
            cands = []
            for x in ordered(s):
                e2 = dict(env)
                e2[n[1]] = x
                if self.truth(self.ev(n[3], e2)):
                    cands.append(x)
            if not cands:
                raise EvalError("CHOOSE: no element satisfies the predicate")
            if len(cands) > 1:
                self.choose_log.append(len(cands))
            return cands[self.choose_pick % len(cands)]
        if k == "unchanged":
            return all(self.sp is not None and self.sp.get(v, _MISSING) == self.s[v] for v in self.unchanged_vars(n[1]))
        if k == "subset":
            s = ordered(self.ev(n[1], env))
            return frozenset(frozenset(x for i, x in enumerate(s) if (mask >> i) & 1) for mask in range(1 << len(s)))
        if k == "bigunion":
            out = set()
            for x in self.ev(n[1], env):
                out |= x
            return frozenset(out)
        raise EvalError("cannot evaluate %s" % k)

    @staticmethod
    def truth(v):
        if v is True or v is False:
            return v
        raise EvalError("not a boolean: %r" % (v,))

    def binop(self, op, a, b, env):
        if op == "/\\":
            return self.truth(self.ev(a, env)) and self.truth(self.ev(b, env))
        if op == "\\/":
            return self.truth(self.ev(a, env)) or self.truth(self.ev(b, env))
        if op == "=>":
            return (not self.truth(self.ev(a, env))) or self.truth(self.ev(b, env))
        x, y = self.ev(a, env), self.ev(b, env)
        if op == "=":
            return x == y
        if op in ("#", "/="):
            return x != y
        if op == "<=>":
            return self.truth(x) == self.truth(y)
        if op in ("<", ">", "<=", "=<", ">=", "+", "-", "*", "%", "\\div", ".."):
            for v in (x, y):
                if not isinstance(v, int) or isinstance(v, bool):
                    raise EvalError("arithmetic on a non-number: %s %s %s" % (fmt(x), op, fmt(y)))
            if op == "<":
                return x < y
            if op == ">":
                return x > y
            if op in ("<=", "=<"):
                return x <= y
            if op == ">=":
                return x >= y
            if op == "+":
                return x + y
            if op == "-":
                return x - y
            if op == "*":
                return x * y
            if op == "%":
                return x % y
            if op == "\\div":
                return x // y
            return frozenset(range(x, y + 1))
        if op == "\\in":
            return x in y
        if op == "\\notin":
            return x not in y
        if op == "\\subseteq":
            return x <= y
        if op in ("\\union", "\\cup"):
            return x | y
        if op in ("\\cap", "\\intersect"):
            return x & y
        if op == "\\":
            return x - y
        if op == "@@":
            d = dict(y.d)
            d.update(x.d)
            return Fn(d)
        if op == ":>":
            return Fn({x: y})
        if op == "\\o":
            return seq([x.d[i] for i in range(1, len(x.d) + 1)] + [y.d[i] for i in range(1, len(y.d) + 1)])
        raise EvalError("operator %s" % op)

    def except_one(self, f, path, rhs, env):
        kind, key = path[0]
        keyv = self.ev(key, env) if kind == "idx" else key
        if not isinstance(f, Fn) or keyv not in f.d:
            raise EvalError("EXCEPT: %s is not in the domain" % (fmt(keyv) if kind == "idx" else keyv))
        old = f.d[keyv]
        if len(path) == 1:
            e2 = dict(env)
            e2["@"] = old
            new = self.ev(rhs, e2)
        else:
            new = self.except_one(old, path[1:], rhs, env)
        d = dict(f.d)
        d[keyv] = new
        return Fn(d)

    # ---- actions (TLC's way of finding the next states)
    def unchanged_vars(self, n):
        if n[0] == "tuple":
            out = []
            for x in n[1]:
                out += self.unchanged_vars(x)
            return out
        if n[0] == "id":
            if n[1] in self.varset:
                return [n[1]]
            if n[1] in self.m.defs:
                return self.unchanged_vars(self.m.body(n[1])[1])
        raise EvalError("UNCHANGED of something that is not a tuple of variables")

    def has_prime(self, n):
        """does evaluating n (definitions expanded) involve a primed variable?"""
        key = id(n)
        r = self._primed.get(key)
        if r is not None:
            return r
        self._primed[key] = False  # cycle guard
        hp, k = self.has_prime, n[0]
        if k in ("prime", "unchanged"):
            r = True
        elif k in ("lit", "at", "typeexpr"):
            r = False
        elif k == "id":
            r = n[1] in self.m.defs and hp(self.m.body(n[1])[1])
        elif k == "call":
            r = (n[1] in self.m.defs and hp(self.m.body(n[1])[1])) or any(hp(a) for a in n[2])
        elif k == "bin":
            r = hp(n[2]) or hp(n[3])
        elif k in ("and", "or", "tuple", "setenum"):
            r = any(hp(x) for x in n[1])
        elif k in ("not", "neg", "domain", "subset", "bigunion"):
            r = hp(n[1])
        elif k == "if":
            r = hp(n[1]) or hp(n[2]) or hp(n[3])
        elif k == "let":
            r = any(hp(body) for _, _, body in n[1]) or hp(n[2])
        elif k == "app":
            r = hp(n[1]) or hp(n[2])
        elif k == "dot":
            r = hp(n[1])
        elif k == "record":
            r = any(hp(e) for _, e in n[1])
        elif k == "setfilter":
            r = hp(n[2]) or hp(n[3])
        elif k == "setmap":
            r = hp(n[1]) or any(hp(sx) for _, sx in n[2])
        elif k in ("fcons", "exists", "forall"):
            r = any(hp(sx) for _, sx in n[1]) or hp(n[2])
        elif k == "except":
            r = hp(n[1]) or any(hp(rhs) or any(kind == "idx" and hp(key_) for kind, key_ in path) for path, rhs in n[2])
        elif k == "choose":
            r = hp(n[2]) or hp(n[3])
        elif k == "lambda":
            r = hp(n[2])
        else:
            raise EvalError("has_prime: %s" % k)
        self._primed[key] = r
        return r

    def gen(self, n, env, sp):
        """yield every completion of the partial next state sp that makes formula n true"""
        k = n[0]
        if k == "and" or (k == "bin" and n[1] == "/\\"):
            items = n[1] if k == "and" else [n[2], n[3]]

            def rec(i, cur):
                if i == len(items):
                    yield cur
                    return
                for nxt in self.gen(items[i], env, cur):
                    yield from rec(i + 1, nxt)
            yield from rec(0, sp)
            return
        if k == "or" or (k == "bin" and n[1] == "\\/"):
            for it in (n[1] if k == "or" else [n[2], n[3]]):
                yield from self.gen(it, env, sp)
            return
        if not self.has_prime(n) and not (k in ("id", "call") and self.local_has_prime(n, env)):
            self.sp = sp
            if self.truth(self.ev(n, env)):
                yield sp
            return
        if k == "exists":
            for e2, _ in self.bindings(n[1], env):
                yield from self.gen(n[2], e2, sp)
            return
        if k == "if":
            self.sp = sp
            yield from self.gen(n[2] if self.truth(self.ev(n[1], env)) else n[3], env, sp)
            return
        if k == "let":
            e2 = dict(env)
            for name, params, body in n[1]:
                e2[name] = Closure(params, body, e2)
            yield from self.gen(n[2], e2, sp)
            return
        if k == "unchanged":
            cur = sp
            for v in self.unchanged_vars(n[1]):
                if v in cur:
                    if cur[v] != self.s[v]:
                        return
                else:
                    cur = dict(cur)
                    cur[v] = self.s[v]
            yield cur
            return
        if k == "bin" and n[1] in ("=", "\\in") and n[2][0] == "prime" and n[2][1][0] == "id" and n[2][1][1] in self.varset:
            var = n[2][1][1]
            self.sp = sp
            val = self.ev(n[3], env)
            if n[1] == "=":
                if var in sp:
                    if sp[var] == val:
                        yield sp
                else:
                    cur = dict(sp)
                    cur[var] = val
                    yield cur
            else:
                for x in ordered(val):
                    if var in sp:
                        if sp[var] == x:
                            yield sp
                    else:
                        cur = dict(sp)
                        cur[var] = x
                        yield cur
            return
        if k in ("id", "call"):
            name = n[1]
            if name in env and isinstance(env[name], Closure):
                clo = env[name]
            elif name in self.m.defs:
                params, body = self.m.body(name)
                clo = Closure(params, body, {})
            else:
                raise EvalError("action %s is not defined" % name)
            self.sp = sp
            args = [self.ev(a, env) for a in (n[2] if k == "call" else [])]
            e2 = dict(clo.env)
            e2.update(zip(clo.params, args))
            yield from self.gen(clo.body, e2, sp)
            return
        # anything else that mentions a primed variable: a test on a determined next state
        self.sp = sp
        if self.truth(self.ev(n, env)):
            yield sp

    def local_has_prime(self, n, env):
        v = env.get(n[1])
        return isinstance(v, Closure) and self.has_prime(v.body)

    # ---- the three things a model checker asks
    def initial_states(self, init="Init"):
        """Init is a conjunction of `variable = value` (VSR.tla:323-348): evaluate it the same way, with the unprimed
        variables as the unknowns"""
        params, body = self.m.body(init)
        self.s = {}
        st = {}

        def walk(n, env):
            if n[0] == "let":
                e2 = dict(env)
                for name, ps, b in n[1]:
                    e2[name] = Closure(ps, b, e2)
                walk(n[2], e2)
            elif n[0] == "and":
                for it in n[1]:
                    walk(it, env)
            elif n[0] == "bin" and n[1] == "=" and n[2][0] == "id" and n[2][1] in self.varset and n[2][1] not in st:
                st[n[2][1]] = self.ev(n[3], env)
                self.s = st
            else:
                if not self.truth(self.ev(n, env)):
                    raise EvalError("Init is not satisfiable the simple way")
        walk(body, {})
        missing = [v for v in self.m.variables if v not in st]
        if missing:
            raise EvalError("Init leaves %s undetermined" % missing)
        return [dict(st)]

    def successors(self, state, next_name="Next"):
        """[(action name, next state)] for every way Next can be satisfied from `state`, duplicates kept (TLC's
        'states generated' counts them)"""
        self.s = state
        params, body = self.m.body(next_name)
        disj = body[1] if body[0] == "or" else [body]
        out = []
        for d in disj:
            label = d[1] if d[0] == "id" else "?"
            for sp in self.gen(d, {}, {}):
                missing = [v for v in self.m.variables if v not in sp]
                if missing:
                    raise EvalError("%s leaves %s undetermined" % (label, missing))
                out.append((label, sp))
        self.sp = None
        return out

    def holds(self, name, state):
        self.s, self.sp = state, None
        return self.truth(self.lookup(name, {}))

    def project(self, state, name="view"):
        self.s, self.sp = state, None
        return self.lookup(name, {})


_MISSING = object()


def _seq_items(f):
    if not isinstance(f, Fn) or not f.is_seq():
        raise EvalError("not a sequence: %s" % fmt(f))
    return [f.d[i] for i in range(1, len(f.d) + 1)]


BUILTINS = {
    "Cardinality": lambda ev, s: len(s),
    "Len": lambda ev, f: len(_seq_items(f)),
    "Append": lambda ev, f, x: seq(_seq_items(f) + [x]),
    "Head": lambda ev, f: _seq_items(f)[0],
    "Tail": lambda ev, f: seq(_seq_items(f)[1:]),
    "SubSeq": lambda ev, f, a, b: seq(_seq_items(f)[a - 1:b]),
    "Quantify": lambda ev, s, clo: sum(1 for x in s if ev.truth(ev.apply_closure(clo, [x]))),
    "Permutations": lambda ev, s: frozenset(Fn(dict(zip(ordered(s), p))) for p in permutations(ordered(s))),
}


# ------------------------------------------------------------------------------------------------ convenience


class _NoModule:
    defs, variables, constants = {}, [], []


class _ModelValues(dict):
    """constants of a printed value: every bare identifier is a model value (Normal, v1, PrepareMsg, Nil, ...)"""

    def __missing__(self, k):
        return ModelValue(k)

    def __contains__(self, k):
        return True


def parse_state_record(text):
    """a state printed as `var |-> value, ...` lines (the oracle's and the product's printers; TLC's dumpTrace records)
    -> dict variable -> value"""
    ev = Evaluator(_NoModule(), _ModelValues())
    ev.c = _ModelValues()
    return dict(ev.ev(parse_expression("[" + text.strip().rstrip(",") + "]"), {}).d)


def load_vsr(path, R, C, values, L, restart=0):
    """the module at `path` bound to the constants of a VSR.cfg (VSR.cfg:3-24: numbers, a set of model values, X = X)"""
    m = Module(open(path).read())
    consts = {"ReplicaCount": R, "ClientCount": C, "Values": frozenset(ModelValue(v) for v in values),
              "StartViewOnTimerLimit": L, "RestartEmptyLimit": restart}
    for name in m.constants:
        if name not in consts:
            consts[name] = ModelValue(name)
    return Evaluator(m, consts)


def bfs(ev, view="view", invariant=None, max_depth=0, max_states=0, keep_levels=True):
    """TLC-style breadth-first search straight from the module text: states are identified by their VIEW value (first
    arrival represents the class, as in TLC), every successor found counts as generated.  No symmetry reduction.
    `invariant`: a definition name or a list of them, evaluated on every new state.
    Returns dict(level_sizes, level_generated, generated, distinct, depth, violation_depth, levels=[[state, ...], ...])."""
    init = ev.initial_states()
    seen = set()
    frontier = []
    for st in init:
        k = ev.project(st, view) if view else Fn(dict(st))
        if k not in seen:
            seen.add(k)
            frontier.append(st)
    out = dict(level_sizes=[len(frontier)], level_generated=[], generated=len(init), distinct=len(frontier), depth=1, violation_depth=0,
               levels=[list(frontier)], ambiguous_choose=0, deadlock_depth=0)
    invs = [invariant] if isinstance(invariant, str) else list(invariant or ())
    if any(not ev.holds(i, st) for st in frontier for i in invs):
        out["violation_depth"] = 1
    while frontier and not (max_depth and out["depth"] >= max_depth) and not (max_states and out["distinct"] >= max_states):
        nxt, gen = [], 0
        for st in frontier:
            ev.choose_log = []
            succ = ev.successors(st)
            if not succ and not out["deadlock_depth"]:
                out["deadlock_depth"] = out["depth"]  # TLC's "deadlock": a state Next cannot leave
            for _, sp in succ:
                gen += 1
                k = ev.project(sp, view) if view else Fn(dict(sp))
                if k not in seen:
                    seen.add(k)
                    nxt.append(sp)
                    if invs and not out["violation_depth"] and not all(ev.holds(i, sp) for i in invs):
                        out["violation_depth"] = out["depth"] + 1
            out["ambiguous_choose"] += 1 if ev.choose_log else 0
        out["level_generated"].append(gen)
        out["generated"] += gen
        if not nxt:
            break
        out["level_sizes"].append(len(nxt))
        if keep_levels:
            out["levels"].append(nxt)
        out["distinct"] += len(nxt)
        out["depth"] += 1
        frontier = nxt
    return out
