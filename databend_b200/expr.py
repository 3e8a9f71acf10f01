"""Tiny expression builder producing the flattened SelectExpr tree (dbx_predicate).

Mirrors how the reference lowers a filter `Expr` into `SelectExpr`
(src/query/expression/src/filter/select_expr.rs:34-50, SelectExprBuilder :80-330):
And / Or / Compare(op, lhs, rhs) / BooleanColumn / BooleanScalar, where a Compare operand is
a column ref, a literal, or one scalar call `column % literal`
(src/query/functions/src/scalars/numeric_basic_arithmetic/src/arithmetic_modulo.rs:29-97).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional, Union

from . import abi
from .block import make_scalar


@dataclass
class ColumnRef:
    index: int
    arith: int = abi.ARITH_NONE
    arith_const: Optional["Literal"] = None

    def __mod__(self, other: "Literal") -> "ColumnRef":
        assert self.arith == abi.ARITH_NONE
        return ColumnRef(self.index, abi.ARITH_MODULO, other)


@dataclass
class Literal:
    value: object
    dtype: int


def col(index: int) -> ColumnRef:
    return ColumnRef(index)


def lit(value, dtype: Optional[int] = None) -> Literal:
    """Integer literals bind to the smallest type like the reference's constant folder
    (`3` is UInt8: SURVEY a3)."""
    if dtype is None:
        if isinstance(value, float):
            dtype = abi.F64
        elif value is None:
            dtype = abi.U8
        elif value >= 0:
            dtype = abi.U8 if value < 2**8 else abi.U16 if value < 2**16 else abi.U32 if value < 2**32 else abi.U64
        else:
            dtype = abi.I8 if value >= -2**7 else abi.I16 if value >= -2**15 else abi.I32 if value >= -2**31 else abi.I64
    return Literal(value, dtype)


Operand = Union[ColumnRef, Literal]


@dataclass
class Node:
    kind: int
    cmp: int = 0
    lhs: Optional[Operand] = None
    rhs: Optional[Operand] = None
    children: Optional[List["Node"]] = None
    value: int = 0


def compare(op: int, lhs: Operand, rhs: Operand) -> Node:
    """An operand may also be a numeric scalar_expr.SExpr: the operator evaluates it as a computed column."""
    return Node(abi.PRED_CMP, cmp=op, lhs=lhs, rhs=rhs)


def eq(a, b): return compare(abi.EQ, a, b)
def ne(a, b): return compare(abi.NE, a, b)
def lt(a, b): return compare(abi.LT, a, b)
def le(a, b): return compare(abi.LE, a, b)
def gt(a, b): return compare(abi.GT, a, b)
def ge(a, b): return compare(abi.GE, a, b)


def and_(*children: Node) -> Node:
    return Node(abi.PRED_AND, children=list(children))


def or_(*children: Node) -> Node:
    return Node(abi.PRED_OR, children=list(children))


def bool_column(index) -> Node:
    """A Boolean input column, or a Boolean scalar_expr.SExpr (a computed column)."""
    return Node(abi.PRED_BOOLCOL, value=index)


def bool_scalar(v: bool) -> Node:
    return Node(abi.PRED_CONST, value=int(v))


def _operand(o: Operand, computed=None) -> abi.Operand:
    c = abi.Operand()
    if not isinstance(o, (Literal, ColumnRef)):  # scalar_expr.SExpr: its computed column
        c.is_const = 0
        c.col = _computed_col(o, computed)
        return c
    if isinstance(o, Literal):
        c.is_const = 1
        c.c = make_scalar(o.dtype, o.value)
    else:
        c.is_const = 0
        c.col = o.index
        c.arith = o.arith
        if o.arith != abi.ARITH_NONE:
            c.c = make_scalar(o.arith_const.dtype, o.arith_const.value)
    return c


def _computed_col(e, computed) -> int:
    if computed is None:
        raise ValueError("a predicate with scalar expressions needs the operator's computed-column list")
    return computed.column(e)


def sexprs(root: Optional[Node]):
    """The scalar expressions (computed columns) a predicate uses, in order."""
    if root is None:
        return []
    out = []
    if root.kind == abi.PRED_CMP:
        out += [o for o in (root.lhs, root.rhs) if not isinstance(o, (Literal, ColumnRef))]
    elif root.kind == abi.PRED_BOOLCOL and not isinstance(root.value, int):
        out.append(root.value)
    for ch in root.children or []:
        out += sexprs(ch)
    return out


def build_predicate(root: Optional[Node], computed=None) -> abi.Predicate:
    """Post-order flattening into dbx_predicate.  `computed` (scalar_expr.Computed) numbers the
    scalar expressions the predicate uses."""
    p = abi.Predicate()
    p.n_nodes = 0
    if root is None:
        return p
    out: List[abi.PredNode] = []

    def emit(n: Node):
        if n.kind in (abi.PRED_AND, abi.PRED_OR):
            assert len(n.children) >= 2
            for ch in n.children:
                emit(ch)
        pn = abi.PredNode()
        pn.kind = n.kind
        pn.cmp = n.cmp
        pn.value = n.value if isinstance(n.value, int) else _computed_col(n.value, computed)
        if n.kind == abi.PRED_CMP:
            pn.lhs = _operand(n.lhs, computed)
            pn.rhs = _operand(n.rhs, computed)
        if n.children:
            pn.n_children = len(n.children)
        out.append(pn)

    emit(root)
    if len(out) > abi.MAX_PRED_NODES:
        raise ValueError("predicate too large for dbx_predicate")
    for i, pn in enumerate(out):
        p.nodes[i] = pn
    p.n_nodes = len(out)
    return p
