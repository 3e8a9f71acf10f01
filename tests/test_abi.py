"""The C-ABI library loads on a CPU-only box, exports every symbol include/dbx.h declares,
and FAILS LOUDLY (no CPU fallback) when there is no GPU.  No compute calls are made here."""
import ctypes as C
import os
import re

import pytest

from databend_b200 import abi, build, lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_builds_and_exports_every_declared_symbol():
    so = build.build()
    assert os.path.exists(so)
    L = lib.load()
    with open(os.path.join(ROOT, "include", "dbx.h")) as f:
        header = f.read()
    declared = set(re.findall(r"^(?:int32_t|int64_t|const char\*)\s+(dbx_[a-z0-9_]+)\s*\(", header, flags=re.M))
    assert declared, "no declarations parsed"
    for name in sorted(declared):
        assert hasattr(L, name), f"libdbx.so does not export {name}"
    assert set(abi.EXPORTS) == declared, set(abi.EXPORTS) ^ declared
    assert L.dbx_abi_version() == abi.ABI_VERSION


def test_struct_layouts_match_header_expectations():
    # natural-alignment layouts of include/dbx.h (x86-64 / aarch64 LP64)
    assert C.sizeof(abi.Scalar) == 16
    assert C.sizeof(abi.Column) == 80
    assert C.sizeof(abi.Block) == 40
    assert C.sizeof(abi.Operand) == 32
    assert C.sizeof(abi.PredNode) == 80
    assert C.sizeof(abi.Predicate) == 8 + 16 * 80
    assert C.sizeof(abi.AggDesc) == 8


def test_no_gpu_means_loud_failure_not_cpu_fallback():
    L = lib.load()
    n = C.c_int32(-1)
    st = L.dbx_device_count(C.byref(n))
    if st == abi.OK:
        pytest.skip("a GPU is present")
    assert st == abi.ERR_NO_DEVICE
    with pytest.raises(lib.DbxError) as ei:
        lib.require_device()
    assert "no CPU fallback" in str(ei.value)
    # operator creation must fail too
    from databend_b200.transforms import AggregatorParams, TransformPartialAggregate
    with pytest.raises(lib.DbxError):
        TransformPartialAggregate(AggregatorParams([0], [("sum", 1)]), [abi.I64, abi.I64])


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "databend_b200")
    for dirpath, _, files in os.walk(pkg):
        for fn in files:
            if fn.endswith((".py", ".cu", ".cuh", ".h", ".cc")):
                with open(os.path.join(dirpath, fn)) as f:
                    src = f.read()
                for pat in (r"^\s*(from|import)\s+oracle", r"libdbx_oracle", r"dbx_oracle\.h", r"\borc_[a-z_]+\s*\("):
                    assert not re.search(pat, src, flags=re.M), f"{fn} uses the oracle ({pat})"


def test_ctypes_mirror_matches_the_header_field_by_field(tmp_path):
    """Compile a probe against include/dbx.h with the system C compiler and compare sizeof / offsetof
    of every struct that crosses the ABI with the ctypes mirror in databend_b200/abi.py."""
    import subprocess
    structs = {
        "dbx_scalar": (abi.Scalar, ["dtype", "is_null", "v"]),
        "dbx_column": (abi.Column, ["dtype", "mem", "is_const", "vec_dim", "len", "data", "data_bit_offset", "validity",
                                    "validity_bit_offset", "null_count", "konst"]),
        "dbx_block": (abi.Block, ["num_rows", "num_cols", "cols", "meta", "owner"]),
        "dbx_operand": (abi.Operand, ["is_const", "col", "arith", "c"]),
        "dbx_pred_node": (abi.PredNode, ["kind", "cmp", "n_children", "value", "lhs", "rhs"]),
        "dbx_predicate": (abi.Predicate, ["n_nodes", "nodes"]),
        "dbx_agg_desc": (abi.AggDesc, ["kind", "arg_col"]),
        "dbx_agg_params": (abi.AggParams, ["n_group_cols", "group_cols", "n_aggs", "aggs", "filter", "expected_groups"]),
        "dbx_topk_params": (abi.TopkParams, ["key_col", "asc", "nulls_first", "limit", "n_extra_keys", "extra_key_cols", "extra_asc", "extra_nulls_first"]),
        "dbx_join_params": (abi.JoinParams, ["kind", "build_key_col", "probe_key_col", "n_build_cols", "expected_build_rows"]),
        "dbx_expr_node": (abi.ExprNode, ["kind", "func", "col", "cast_to", "try_cast", "c"]),
        "dbx_expr": (abi.Expr, ["n_nodes", "nodes"]),
    }
    lines = ['#include <stdio.h>', '#include <stddef.h>', f'#include "{os.path.join(ROOT, "include", "dbx.h")}"', "int main(void) {"]
    for cname, (_, fields) in structs.items():
        lines.append(f'  printf("{cname} %zu\\n", sizeof({cname}));')
        for f in fields:
            lines.append(f'  printf("{cname}.{f} %zu\\n", offsetof({cname}, {f}));')
    lines += ["  return 0;", "}"]
    src = tmp_path / "probe.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "probe"
    subprocess.check_call(["gcc", "-std=c11", "-o", str(exe), str(src)])
    out = dict(l.split() for l in subprocess.check_output([str(exe)], text=True).splitlines())
    for cname, (ctype, fields) in structs.items():
        assert int(out[cname]) == C.sizeof(ctype), cname
        for f in fields:
            assert int(out[f"{cname}.{f}"]) == getattr(ctype, f).offset, f"{cname}.{f}"
    # enum values the Python side hard-codes
    assert (abi.JOIN_INNER, abi.JOIN_LEFT_SEMI, abi.JOIN_LEFT_ANTI, abi.JOIN_LEFT) == (0, 1, 2, 3)


def test_runtime_specialisation_compiles_here():
    """NVRTC is dlopen'ed by libdbx; the specialised aggregate kernels of a canned plan must compile
    for sm_90a in this image (no GPU involved)."""
    import ctypes as C
    from databend_b200.lib import load
    buf = C.create_string_buffer(4096)
    rc = load().dbx_agg_jit_selftest(buf, 4096)
    assert rc == abi.OK, buf.value.decode()
    rc = load().dbx_eval_jit_selftest(buf, 4096)
    assert rc == abi.OK, buf.value.decode()
