#!/usr/bin/env python
"""Dev-time tool: derive the lifting-network IR of Daala's integer DCTs.

The 1-D transforms of the reference (src/dct.c:87-790 hand-written 4/8/16-point,
src/dct.c:808-4023 nested OD_FDCT_*/OD_FDST_* macros for 32/64-point, functions
od_bin_fdct32 :4219, od_bin_idct32 :4321, od_bin_fdct64 :4422, od_bin_idct64
:4622) are *normative* sequences of integer lifting steps: every
`(t*C + R) >> S` must be evaluated in the reference's order for the output to
be bit-exact.  This script turns each function into a flat, scope-free list of
register operations (our own IR, written to daala_b200/csrc/gen/dct_ir.json).
All code generation (CUDA device functions, the plain-C oracle port) starts
from that IR -- see tools/gen_dct.py.  The reference sources are needed only when the
IR is (re)extracted, never at build or run time.

How: the C preprocessor expands the macro tree (with OD_DCT_RSHIFT kept
symbolic and the overflow-check instrumentation defined away), pycparser
parses each expanded function body, and a small walker renames block-scoped
temporaries to unique registers and flattens do{..}while(0) blocks.
"""
import json
import os
import re
import subprocess
import sys
import tempfile

from pycparser import c_ast, c_parser

REF = os.environ.get("DAALA_REF", os.path.join(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))), "reference"))
OUT = os.path.join(os.path.dirname(__file__), "..", "daala_b200", "csrc", "gen", "dct_ir.json")

PRELUDE = """
#define OD_DCT_OVERFLOW_CHECK(val, scale, offset, idx)
#define OD_DCT_RSHIFT(a, b) __rshift(a, b)
#define OD_COEFF_BITS (32)
#define OD_DISABLE_FILTER (0)
#define OD_DEBLOCKING (0)
#define OD_NBSIZES (5)
"""


def preprocess(path):
    src = open(path).read()
    src = re.sub(r'^\s*#\s*include.*$', '', src, flags=re.M)
    with tempfile.NamedTemporaryFile("w", suffix=".c", delete=False) as f:
        f.write(PRELUDE + src)
        tmp = f.name
    try:
        return subprocess.check_output(["gcc", "-E", "-P", tmp], text=True)
    finally:
        os.unlink(tmp)


def function_text(pp, name):
    m = re.search(r'\bvoid\s+%s\s*\(' % re.escape(name), pp)
    if not m:
        raise KeyError(name)
    i = pp.index('{', m.end())
    depth, j = 0, i
    while True:
        if pp[j] == '{':
            depth += 1
        elif pp[j] == '}':
            depth -= 1
            if depth == 0:
                break
        j += 1
    return pp[m.start():j + 1]


class Flattener:
    """Walks one function body; emits ops over uniquely named registers."""

    def __init__(self, in_name, out_name):
        self.in_name, self.out_name = in_name, out_name
        self.scopes = [{}]
        self.count = {}
        self.ops = []
        self.regs = []
        self.local_arrays = {}

    def declare(self, name):
        n = self.count.get(name, 0)
        self.count[name] = n + 1
        reg = name if n == 0 else "%s_%d" % (name, n)
        self.scopes[-1][name] = reg
        self.regs.append(reg)
        return reg

    def lookup(self, name):
        for s in reversed(self.scopes):
            if name in s:
                return s[name]
        raise KeyError(name)

    def const(self, node):
        """Evaluate an index expression such as `3*xstride` -> 3."""
        if isinstance(node, c_ast.Constant):
            return int(node.value, 0)
        if isinstance(node, c_ast.BinaryOp) and node.op == '*':
            if isinstance(node.right, c_ast.ID) and node.right.name == 'xstride':
                return self.const(node.left)
        if isinstance(node, c_ast.ID) and node.name == 'xstride':
            return 1
        raise ValueError("index: %s" % node)

    def mem_index(self, node):
        """x[k*xstride], *(x + k*xstride), y[k] -> (array, k) or None."""
        if isinstance(node, c_ast.ArrayRef) and isinstance(node.name, c_ast.ID):
            if node.name.name in self.local_arrays:
                return None
            return node.name.name, self.const(node.subscript)
        if isinstance(node, c_ast.UnaryOp) and node.op == '*':
            e = node.expr
            if isinstance(e, c_ast.BinaryOp) and e.op == '+' and isinstance(e.left, c_ast.ID):
                return e.left.name, self.const(e.right)
        return None

    def expr(self, node):
        if isinstance(node, c_ast.ID):
            return self.lookup(node.name)
        if isinstance(node, c_ast.Constant):
            return int(node.value, 0)
        if isinstance(node, c_ast.Cast):
            return self.expr(node.expr)
        if isinstance(node, c_ast.UnaryOp):
            if node.op == '-':
                return ['neg', self.expr(node.expr)]
            if node.op == '*':
                arr, k = self.mem_index(node)
                return ['ld', k]
        if isinstance(node, c_ast.ArrayRef):
            if node.name.name in self.local_arrays:
                return self.local_arrays[node.name.name][self.const(node.subscript)]
            arr, k = self.mem_index(node)
            assert arr == self.in_name, arr
            return ['ld', k]
        if isinstance(node, c_ast.BinaryOp):
            assert node.op in ('+', '-', '*', '>>', '&', '/', '<<'), node.op
            return [node.op, self.expr(node.left), self.expr(node.right)]
        if isinstance(node, c_ast.FuncCall) and node.name.name == '__rshift':
            a, b = node.args.exprs
            assert self.const(b) == 1
            return ['rsh1', self.expr(a)]
        raise ValueError("expr: %r" % node)

    def stmt(self, node):
        if isinstance(node, c_ast.Compound):
            self.scopes.append({})
            for it in node.block_items or []:
                self.stmt(it)
            self.scopes.pop()
        elif isinstance(node, c_ast.DoWhile):
            self.stmt(node.stmt)
        elif isinstance(node, c_ast.Decl):
            assert node.init is None
            if isinstance(node.type, c_ast.ArrayDecl):
                # local scratch array int t[N] -> registers t_0 .. t_{N-1}
                n = int(node.type.dim.value, 0)
                self.local_arrays[node.name] = [self.declare("%s%d" % (node.name, i)) for i in range(n)]
            else:
                self.declare(node.name)
        elif isinstance(node, c_ast.Assignment):
            mem = self.mem_index(node.lvalue)
            if mem is not None:
                arr, k = mem
                assert arr == self.out_name and node.op == '='
                self.ops.append(['st', k, self.expr(node.rvalue)])
                return
            if isinstance(node.lvalue, c_ast.ArrayRef):
                dst = self.local_arrays[node.lvalue.name.name][self.const(node.lvalue.subscript)]
            else:
                dst = self.lookup(node.lvalue.name)
            rhs = self.expr(node.rvalue)
            if node.op == '=':
                self.ops.append(['set', dst, rhs])
            else:
                assert node.op in ('+=', '-='), node.op
                self.ops.append(['set', dst, [node.op[0], dst, rhs]])
        elif isinstance(node, c_ast.EmptyStatement):
            pass
        else:
            raise ValueError("stmt: %r" % node)


def extract(pp, name, in_name, out_name):
    text = function_text(pp, name)
    text = re.sub(r'\b_([xy])\b', r'\1', text)  # filter.c spells its arguments _x / _y
    text = "typedef int od_coeff;\n" + text
    ast = c_parser.CParser().parse(text)
    fn = [e for e in ast.ext if isinstance(e, c_ast.FuncDef)][0]
    fl = Flattener(in_name, out_name)
    fl.stmt(fn.body)
    return {"regs": fl.regs, "ops": fl.ops}


def main():
    pp = preprocess(os.path.join(REF, "src", "dct.c"))
    ir = {"_comment": "lifting-network IR derived from xiph/daala src/dct.c by "
          "tools/extract_lifting_ir.py; ops: ['set', reg, expr] | ['st', idx, expr]; "
          "expr: reg | int | ['ld', idx] | ['+'|'-'|'*'|'>>', a, b] | ['rsh1', a] "
          "(rsh1(a) = (a + (a < 0)) >> 1, src/filter.h:38-41) | ['neg', a]"}
    for n in (4, 8, 16, 32, 64):
        ir["fdct%d" % n] = extract(pp, "od_bin_fdct%d" % n, "x", "y")
        ir["idct%d" % n] = extract(pp, "od_bin_idct%d" % n, "y", "x")
        print("n=%d: fdct %d ops / %d regs, idct %d ops / %d regs" % (
            n, len(ir["fdct%d" % n]["ops"]), len(ir["fdct%d" % n]["regs"]),
            len(ir["idct%d" % n]["ops"]), len(ir["idct%d" % n]["regs"])), file=sys.stderr)
    # larger lapping filters of src/filter.c (dead in the codec, kept for ABI completeness):
    # od_pre_filter8 :279, od_post_filter8 :366, 16 :519/:678, 32 :852/:1146
    fpp = preprocess(os.path.join(REF, "src", "filter.c"))
    for n in (8, 16, 32):
        ir["prefilter%d" % n] = extract(fpp, "od_pre_filter%d" % n, "x", "y")
        ir["postfilter%d" % n] = extract(fpp, "od_post_filter%d" % n, "y", "x")
        print("filter n=%d: pre %d ops, post %d ops" % (n, len(ir["prefilter%d" % n]["ops"]),
                                                        len(ir["postfilter%d" % n]["ops"])), file=sys.stderr)
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    with open(OUT, "w") as f:
        json.dump(ir, f, separators=(",", ":"))
        f.write("\n")


if __name__ == "__main__":
    main()
