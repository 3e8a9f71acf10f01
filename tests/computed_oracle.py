"""Reference for computed columns: Filter -> EvalScalar -> Aggregate composed from pieces the suite
already trusts: oracle.filter_select on the block (the predicate's computed operands evaluated first;
they cannot raise), eval_oracle.evaluate of every other expression on the SELECTED rows, then
oracle.filter_group_agg over the block extended by the computed columns.  eval_oracle evaluates row by
row in Python: keep blocks to about 1e5 rows."""
import numpy as np

from databend_b200 import abi, expr as E, scalar_expr as S
from databend_b200.block import Column, DataBlock

NAME = {abi.I8: "I8", abi.I16: "I16", abi.I32: "I32", abi.I64: "I64", abi.U8: "U8", abi.U16: "U16", abi.U32: "U32", abi.U64: "U64",
        abi.F32: "F32", abi.F64: "F64", abi.BOOL: "BOOL"}
DT = {v: k for k, v in NAME.items()}
NP = {"I8": np.int8, "I16": np.int16, "I32": np.int32, "I64": np.int64, "U8": np.uint8, "U16": np.uint16, "U32": np.uint32, "U64": np.uint64,
      "F32": np.float32, "F64": np.float64, "BOOL": bool}
FN = {v: k for k, v in S.FUNCS.items()}


def to_tuple(e: S.SExpr):
    """SExpr -> the eval_oracle tree (the form test_eval_gpu.py's to_tuple produces)."""
    if e.kind == abi.EXPR_COLUMN:
        return ("col", e.col)
    if e.kind == abi.EXPR_CONST:
        return ("lit", e.value, NAME[e.dtype])
    if e.kind == abi.EXPR_CAST:
        return ("cast", to_tuple(e.args[0]), NAME[e.dtype], int(e.try_cast))
    return ("call", e.func) + tuple(to_tuple(a) for a in e.args)


class OracleEvalError(Exception):
    def __init__(self, msg, row):
        super().__init__(msg)
        self.msg, self.row = msg, row


def _plain(col: Column, t: int, rows: np.ndarray) -> Column:
    """Rows of a column as a materialised column (Const entries expanded), validity as the schema says."""
    nullable = bool(t & abi.NULLABLE)
    vals, valid = col.values()[rows], col.valid_mask()[rows]
    return Column.from_data(np.asarray(vals, dtype=NP[NAME[t & 0xFF]]), t & 0xFF, validity=valid if nullable else None)


def _eval_columns(cols, types):
    out = []
    for c, t in zip(cols, types):
        out.append((NAME[t & 0xFF], c.values(), c.valid_mask() if t & abi.NULLABLE else None))
    return out


def _computed_column(e, cols, types, rows_of=None):
    from oracle import eval_oracle
    try:
        t, nullable, vals, oks = eval_oracle.evaluate(to_tuple(e), _eval_columns(cols, types))
    except eval_oracle.EvalFailure as f:
        raise OracleEvalError(f.msg, int(rows_of[f.row]) if rows_of is not None else f.row)
    col = Column.from_data(np.asarray(vals, dtype=NP[t]), DT[t], validity=np.asarray(oks, dtype=bool) if nullable else None)
    return col, DT[t] | (abi.NULLABLE if nullable else 0)


def composed(blk: DataBlock, types, params, filt=None, threads=4):
    """-> (oracle result of filter_group_agg, types of the computed columns)."""
    from oracle import oracle as orc
    n_in = len(types)
    comp = params.computed(n_in, filt)
    pred_keys = {S.key(e) for e in E.sexprs(filt)}
    n = blk.num_rows
    all_rows = np.arange(n)
    inputs = [_plain(c, t, all_rows) for c, t in zip(blk.columns, types)]
    ctypes_ = [abi.U8] * len(comp.exprs)
    pred_cols = {}
    for i, e in enumerate(comp.exprs):
        if S.key(e) in pred_keys:
            pred_cols[i], ctypes_[i] = _computed_column(e, inputs, types)
    dummy = Column.from_data(np.zeros(n, dtype=np.uint8), abi.U8)
    if filt is not None:
        blk_a = DataBlock(inputs + [pred_cols.get(i, dummy) for i in range(len(comp.exprs))], n)
        sel = orc.filter_select(blk_a, E.build_predicate(filt, comp)).astype(np.int64)
    else:
        sel = all_rows
    sel_inputs = [_plain(c, t & 0xFF | (t & abi.NULLABLE), sel) for c, t in zip(inputs, types)]
    cols = []
    for i, e in enumerate(comp.exprs):
        if i in pred_cols:
            c = pred_cols[i]
            cols.append(_plain(c, ctypes_[i], sel))
        else:
            c, ctypes_[i] = _computed_column(e, sel_inputs, types, sel)
            cols.append(c)
    blk_b = DataBlock(sel_inputs + cols, len(sel))
    return orc.filter_group_agg(blk_b, params.to_c(None, comp), threads=threads), ctypes_
