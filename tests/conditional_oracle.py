"""CPU reference for conditional expressions (test infrastructure only — never imported by the product).

Extends oracle/eval_oracle.py, which restates the reference's numeric / boolean functions row by row, with
the two nodes whose evaluation is not a plain function of their evaluated arguments (paths relative to the
databend source tree):
  if (lazy)         src/query/expression/src/evaluator.rs:1702-1790 (eval_if): a condition is evaluated only on
                    rows no earlier condition took, a branch only on rows its condition took (a NULL condition
                    counts as false), so a call raises only on rows that reach it.  Signature
                    src/query/functions/src/scalars/control.rs:36-108: condition Boolean NULL, branches and result
                    one type T0, nullable when a branch is.
  assume_not_null   src/query/functions/src/scalars/other.rs:217-229: drops the validity; under a NULL the value
                    is unspecified — the type's default here, as for a NULL scalar.
Every other node goes to eval_oracle with its arguments already evaluated (in program order, so the first
failing call is the same), passed as typed literals.  `composed` is tests/computed_oracle.py's
Filter -> EvalScalar -> Aggregate reference with this evaluator."""
import numpy as np

from oracle import eval_oracle as eo
import computed_oracle as co

EvalFailure = eo.EvalFailure


def _args(e):
    if e[0] == "call":
        return list(e[2:])
    if e[0] == "cast":
        return [e[1]]
    return []


def _rebuild(e, args):
    if e[0] == "call":
        return ("call", e[1]) + tuple(args)
    return ("cast", args[0], e[2], e[3])


def infer(e, col_types):
    """-> (type name, nullable), the trees of eval_oracle plus ("call", "if", c, t, e) and ("call", "assume_not_null", x)."""
    if e[0] in ("col", "lit"):
        return eo.infer(e, col_types)
    args = [infer(a, col_types) for a in _args(e)]
    if e[0] == "call" and e[1] == "if":
        (tc, _), (tt, nt), (te, ne) = args
        if tc != "BOOL" or tt != te:
            raise ValueError("if(): the condition must be Boolean and both branches of one type")
        return (tt, nt or ne)
    if e[0] == "call" and e[1] == "assume_not_null":
        return (args[0][0], False)
    return eo.infer(_rebuild(e, [("lit", None if n else 0, t) for t, n in args]), col_types)


def eval_row(e, row, col_types, r):
    """-> (value, valid); raises EvalFailure for a per-row error on a row that reaches the failing call."""
    if e[0] in ("col", "lit"):
        return eo.eval_row(e, row, col_types, r)
    if e[0] == "call" and e[1] == "if":  # lazy: only the taken branch is evaluated (and can raise) on this row
        c, cok = eval_row(e[2], row, col_types, r)
        return eval_row(e[3] if (cok and c) else e[4], row, col_types, r)
    if e[0] == "call" and e[1] == "assume_not_null":
        v, ok = eval_row(e[2], row, col_types, r)
        return (v, True) if ok else ((False if infer(e[2], col_types)[0] == "BOOL" else 0), True)
    lits = []
    for a in _args(e):
        v, ok = eval_row(a, row, col_types, r)
        lits.append(("lit", v if ok else None, infer(a, col_types)[0]))
    return eo.eval_row(_rebuild(e, lits), row, col_types, r)


def evaluate(e, columns):
    """eval_oracle.evaluate with the nodes above: (type, nullable, values, valid); raises EvalFailure at the
    FIRST failing row."""
    col_types = [(t, valid is not None) for t, _, valid in columns]
    t, nullable = infer(e, col_types)
    n = len(columns[0][1]) if columns else 0
    vals, oks = [], []
    for r in range(n):
        row = []
        for ct, v, valid in columns:
            x = v[r]
            x = float(x) if eo.is_float(ct) else (bool(x) if ct == "BOOL" else int(x))
            row.append((x, True if valid is None else bool(valid[r])))
        v, ok = eval_row(e, row, col_types, r)
        vals.append(v if ok else (False if t == "BOOL" else 0))
        oks.append(ok)
    return t, nullable, vals, oks


def _computed_column(e, cols, types, rows_of=None):
    try:
        t, nullable, vals, oks = evaluate(co.to_tuple(e), co._eval_columns(cols, types))
    except EvalFailure as f:
        raise co.OracleEvalError(f.msg, int(rows_of[f.row]) if rows_of is not None else f.row)
    col = co.Column.from_data(np.asarray(vals, dtype=co.NP[t]), co.DT[t], validity=np.asarray(oks, dtype=bool) if nullable else None)
    return col, co.DT[t] | (co.abi.NULLABLE if nullable else 0)


def composed(blk, types, params, filt=None, threads=4):
    """computed_oracle.composed with conditional expressions: -> (oracle result of filter_group_agg, types of
    the computed columns)."""
    from oracle import oracle as orc
    abi, E, S, DataBlock, Column = co.abi, co.E, co.S, co.DataBlock, co.Column
    n_in = len(types)
    comp = params.computed(n_in, filt)
    pred_keys = {S.key(e) for e in E.sexprs(filt)}
    n = blk.num_rows
    all_rows = np.arange(n)
    inputs = [co._plain(c, t, all_rows) for c, t in zip(blk.columns, types)]
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
    sel_inputs = [co._plain(c, t, sel) for c, t in zip(inputs, types)]
    cols = []
    for i, e in enumerate(comp.exprs):
        if i in pred_cols:
            cols.append(co._plain(pred_cols[i], ctypes_[i], sel))
        else:
            c, ctypes_[i] = _computed_column(e, sel_inputs, types, sel)
            cols.append(c)
    blk_b = DataBlock(sel_inputs + cols, len(sel))
    return orc.filter_group_agg(blk_b, params.to_c(None, comp), threads=threads), ctypes_
