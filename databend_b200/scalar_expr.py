"""Scalar expressions over a DataBlock: host-side mirror of the reference's `Expr` tree
(src/query/expression/src/expression.rs: ColumnRef / Constant / Cast / FunctionCall) for the numeric
and boolean functions libdbx evaluates on the device (include/dbx.h: dbx_eval_scalar).  Trees are
flattened to the postfix program the C-ABI takes; no compute happens here."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import List, Optional, Tuple

from . import abi
from .block import Column, DataBlock, make_scalar
from .lib import DbxError, check, load

FUNCS = {"plus": abi.FN_PLUS, "minus": abi.FN_MINUS, "multiply": abi.FN_MULTIPLY, "divide": abi.FN_DIVIDE, "div": abi.FN_DIV,
         "modulo": abi.FN_MODULO, "negate": abi.FN_NEGATE, "eq": abi.FN_EQ, "noteq": abi.FN_NOTEQ, "lt": abi.FN_LT, "lte": abi.FN_LTE,
         "gt": abi.FN_GT, "gte": abi.FN_GTE, "and": abi.FN_AND, "or": abi.FN_OR, "not": abi.FN_NOT, "is_null": abi.FN_IS_NULL,
         "is_not_null": abi.FN_IS_NOT_NULL, "if": abi.FN_IF, "assume_not_null": abi.FN_ASSUME_NOT_NULL}
UNARY = {"negate", "not", "is_null", "is_not_null", "assume_not_null"}


@dataclass
class SExpr:
    kind: int
    func: str = ""
    col: int = 0
    dtype: int = 0
    value: object = None
    try_cast: bool = False
    args: List["SExpr"] = field(default_factory=list)

    def __add__(self, o): return call("plus", self, o)
    def __sub__(self, o): return call("minus", self, o)
    def __mul__(self, o): return call("multiply", self, o)
    def __truediv__(self, o): return call("divide", self, o)
    def __floordiv__(self, o): return call("div", self, o)
    def __mod__(self, o): return call("modulo", self, o)
    def __neg__(self): return call("negate", self)


def col(i: int) -> SExpr:
    return SExpr(abi.EXPR_COLUMN, col=i)


def lit(value, dtype: int) -> SExpr:
    """Scalar literal of an explicit type (the reference's binder picks the smallest integer type)."""
    return SExpr(abi.EXPR_CONST, dtype=dtype, value=value)


def cast(e: SExpr, dtype: int, try_cast: bool = False) -> SExpr:
    return SExpr(abi.EXPR_CAST, dtype=dtype, try_cast=try_cast, args=[e])


def call(name: str, *args: SExpr) -> SExpr:
    if name not in FUNCS:
        raise DbxError(abi.ERR_UNSUPPORTED, f"function {name} is not built")
    assert len(args) == (1 if name in UNARY else 3 if name == "if" else 2)
    return SExpr(abi.EXPR_CALL, func=name, args=list(args))


# ---- conditionals: the binder's rewrites onto the reference's `if` (paths under
# src/query/sql/src/planner/semantic/type_check/), restated literally.  Branches must already share one
# dtype (add casts as the type checker would); `dtype` names the type of the NULL literal a rewrite adds.
def null(dtype: int) -> SExpr:
    """NULL literal of a branch type."""
    return lit(None, dtype)


def if_(*args: SExpr) -> SExpr:
    """if(c1, r1, ..., cm, rm, else) as m nested ternary IF nodes: if(c1, r1, if(c2, r2, ... else))."""
    assert len(args) >= 3 and len(args) % 2 == 1
    if len(args) == 3:
        return call("if", *args)
    return call("if", args[0], args[1], if_(*args[2:]))


def case_(whens, else_: Optional[SExpr] = None, operand: Optional[SExpr] = None, dtype: Optional[int] = None) -> SExpr:
    """CASE [operand] WHEN c THEN r ... [ELSE e] END (scalar_rewrite.rs:117-142): with an operand each
    condition is eq(operand, c); without ELSE the else is a NULL literal (of `dtype`)."""
    args = []
    for c, r in whens:
        args += [call("eq", operand, c) if operand is not None else c, r]
    if else_ is None:
        assert dtype is not None, "CASE without ELSE: give the branch dtype of its NULL"
        else_ = null(dtype)
    return if_(*args, else_)


def _is_null_literal(e: SExpr) -> bool:
    return e.kind == abi.EXPR_CONST and e.value is None


def coalesce(*args: SExpr, dtype: int) -> SExpr:
    """coalesce(a, b, ...) (special_function.rs:559-606): NULL literals are skipped, every other argument
    becomes is_not_null(a), assume_not_null(a), and the else is NULL."""
    new = []
    for a in args:
        if _is_null_literal(a):
            continue
        new += [call("is_not_null", a), call("assume_not_null", a)]
    new.append(null(dtype))
    if len(new) == 1:
        new += [null(dtype), null(dtype)]
    return if_(*new)


def nullif(x: SExpr, y: SExpr, dtype: int) -> SExpr:
    """nullif(x, y) = if(eq(x, y), NULL, x) (rewrite_function.rs:40-47)."""
    return if_(call("eq", x, y), null(dtype), x)


def iff(c: SExpr, t: SExpr, e: SExpr) -> SExpr:
    """iff(c, t, e) = if(c, t, e) (rewrite_function.rs:66-71)."""
    return if_(c, t, e)


def ifnull(x: SExpr, y: SExpr) -> SExpr:
    """ifnull(x, y) / nvl(x, y) = if(not(is_not_null(x)), y, x) (rewrite_function.rs:72-79)."""
    return if_(call("not", call("is_not_null", x)), y, x)


nvl = ifnull


def nvl2(x: SExpr, y: SExpr, z: SExpr) -> SExpr:
    """nvl2(x, y, z) = if(is_not_null(x), y, z) (rewrite_function.rs:80-86)."""
    return if_(call("is_not_null", x), y, z)


def is_distinct_from(a: SExpr, b: SExpr, not_: bool = False) -> SExpr:
    """a IS [NOT] DISTINCT FROM b (scalar_rewrite.rs:59-89): assume_not_null(if(both NULL, not_, either NULL,
    not not_, a <> b (a = b for NOT)))."""
    def is_null(x):
        return call("not", call("is_not_null", x))
    both = call("and", is_null(a), is_null(b))
    either = call("or", is_null(a), is_null(b))
    compare = call("eq" if not_ else "noteq", a, b)
    return call("assume_not_null", if_(both, lit(not_, abi.BOOL), either, lit(not not_, abi.BOOL), compare))


def flatten(e: SExpr) -> abi.Expr:
    nodes: List[SExpr] = []

    def walk(x: SExpr):
        for a in x.args:
            walk(a)
        nodes.append(x)
    walk(e)
    if len(nodes) > abi.MAX_EXPR_NODES:
        raise DbxError(abi.ERR_UNSUPPORTED, "expression too large")
    out = abi.Expr()
    out.n_nodes = len(nodes)
    for i, x in enumerate(nodes):
        n = out.nodes[i]
        n.kind = x.kind
        if x.kind == abi.EXPR_COLUMN:
            n.col = x.col
        elif x.kind == abi.EXPR_CONST:
            n.c = make_scalar(x.dtype, x.value)
        elif x.kind == abi.EXPR_CAST:
            n.cast_to, n.try_cast = x.dtype, int(x.try_cast)
        else:
            n.func = FUNCS[x.func]
    return out


def key(e: SExpr) -> tuple:
    """Structural identity of an expression (equal keys: one computed column)."""
    return (e.kind, e.func, e.col, e.dtype, repr(e.value), e.try_cast, tuple(key(a) for a in e.args))


class Computed:
    """The distinct expressions an operator evaluates, numbered after its input columns in first-use order
    (column n_inputs + i is exprs[i])."""

    def __init__(self, n_inputs: int):
        self.n_inputs = n_inputs
        self.exprs: List[SExpr] = []
        self._index = {}

    def column(self, e) -> int:
        """Column index of an input index or an SExpr (added on first use)."""
        if not isinstance(e, SExpr):
            return e
        k = key(e)
        if k not in self._index:
            self._index[k] = self.n_inputs + len(self.exprs)
            self.exprs.append(e)
        return self._index[k]

    def to_c(self):
        arr = (abi.Expr * max(1, len(self.exprs)))()
        for i, e in enumerate(self.exprs):
            arr[i] = flatten(e)
        return arr


class EvalError(DbxError):
    def __init__(self, status, message, row):
        super().__init__(status, message)
        self.row = row


def eval_scalar(block: DataBlock, e: SExpr, device: int = 0, out_mem: int = abi.MEM_HOST):
    """Evaluator::run(expr) over `block` -> (result column, its dtype | NULLABLE flag).  With
    out_mem = MEM_DEVICE the result stays in HBM: (library-owned dbx_block to release, dtype)."""
    from .transforms import _block_from_c
    ce = flatten(e)
    b, keep = block.as_c()
    out = abi.Block()
    odt, erow = C.c_int32(0), C.c_int64(-1)
    st = load().dbx_eval_scalar(device, C.byref(ce), C.byref(b), out_mem, C.byref(out), C.byref(odt), C.byref(erow))
    if st != abi.OK:
        msg = (load().dbx_last_error(None) or b"").decode("utf-8", "replace")
        raise EvalError(st, msg, erow.value)
    if out_mem != abi.MEM_HOST:
        return out, odt.value
    res = _block_from_c(out, device)
    return res.columns[0], odt.value
