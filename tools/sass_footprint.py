"""Instruction footprint of the keyframe engine's PVQ kernels (CPU only: nvcc cross-compiles).

Compiles daala_b200/csrc/kf_engine.cu to a cubin with the library's flags (daala_b200/build.py, which
include -lineinfo) and prints, per PVQ kernel: SASS bytes, registers, stack frame, spill bytes and the
STL / LDL / BRA / BSSY / CALL counts.  For one kernel (by default the luma chain kernel
k_pvq_persist<true>) it also splits the bytes by source region, from the line info of every instruction:

  * out-of-line <fn>: the body of a subroutine the kernel calls (a __noinline__ function, or a slow path of
    the CUDA math library), whatever it inlines, found by the subroutine's label;
  * CUDA headers: inlined intrinsics (shuffles, reductions, double-precision math);
  * pvq_math.cuh: the inlined fixed-point helpers;
  * otherwise the innermost function of the project's sources the instruction comes from.

    python tools/sass_footprint.py [--kernel NAME] [--json]
"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from daala_b200 import build as _build  # noqa: E402

SRC = os.path.join(_build.CSRC, "kf_engine.cu")
CUDA_BIN = os.path.dirname(_build.NVCC)
PVQ_KERNELS = ("k_pvq_persist", "k_pvq_split", "k_pvq_prepass", "k_pvq_levels")
COUNTED = ("STL", "LDL", "BRA", "BSSY", "CALL", "WARPSYNC")

def pretty(mangled):
    m = re.search(r"(k_\w+?)I(L[^E]+E(?:L[^E]+E)*)E", mangled)
    if not m:
        m2 = re.search(r"\d+(k_\w+?)E", mangled)
        return m2.group(1) if m2 else mangled
    args = re.findall(r"L(b|i)(\d+)E", m.group(2))
    vals = [("true" if v == "1" else "false") if t == "b" else v for t, v in args]
    return "%s<%s>" % (m.group(1), ", ".join(vals))


def compile_cubin(out_dir):
    cubin = os.path.join(out_dir, "kf_engine.cubin")
    cmd = [_build.NVCC] + _build.FLAGS + ["-Xptxas", "-v", "-cubin", "-o", cubin, SRC]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed:\n%s%s" % (r.stdout, r.stderr))
    return cubin, r.stderr


def parse_ptxas(log):
    """{mangled kernel: {regs, stack, spill_st, spill_ld}} from -Xptxas -v."""
    res, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            cur = res.setdefault(m.group(1), {})
            continue
        if cur is None:
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m:
            cur.update(stack=int(m.group(1)), spill_st=int(m.group(2)), spill_ld=int(m.group(3)))
        m = re.search(r"Used (\d+) registers", line)
        if m:
            cur["regs"] = int(m.group(1))
            cur = None
    return res


def _subroutine(label):
    """Name of an out-of-line subroutine from its label ($kernel$mangled or $__internal_N_$name)."""
    mangled = label.rsplit("$", 1)[-1]
    if not mangled.startswith("_Z"):
        return mangled
    # the last length-prefixed identifier of the mangled name is the function's own
    names = []
    for m in re.finditer(r"(\d+)(?=[A-Za-z_])", mangled):
        names.append(mangled[m.end():m.end() + int(m.group(1))])
    return names[-1] if names else mangled


def disassemble(cubin):
    """{mangled kernel: [(opcode, [(file, line), ...innermost first], subroutine or None)]} from nvdisasm -gi."""
    r = subprocess.run([os.path.join(CUDA_BIN, "nvdisasm"), "-gi", cubin], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvdisasm failed:\n%s" % r.stderr)
    kernels, cur, chain, fresh, sub = {}, None, [], True, None
    for line in r.stdout.splitlines():
        m = re.match(r"\.text\.(\S+):$", line)
        if m:
            cur = kernels.setdefault(m.group(1), [])
            chain, fresh, sub = [], True, None
            continue
        if cur is None:
            continue
        m = re.match(r"(\$\S+):$", line)
        if m:
            sub = _subroutine(m.group(1))
            continue
        m = re.match(r'\s*//## File "([^"]+)", line (\d+)(?: inlined at "([^"]+)", line (\d+))?', line)
        if m:
            if not fresh:
                chain, fresh = [], True
            # each frame line names its call site too; the next line repeats it unless it is the outermost
            for f in ((m.group(1), int(m.group(2))), (m.group(3), int(m.group(4) or 0))):
                if f[0] and (not chain or chain[-1] != f):
                    chain.append(f)
            continue
        m = re.match(r"\s*/\*[0-9a-f]+\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_]*)", line)
        if m:
            cur.append((m.group(1), list(chain), sub))
            fresh = False
    return kernels


_FN_START = re.compile(r"^(?:static\s+)?(?:inline\s+)?(?:__device__|__global__|__host__)[^(]*?(\w+)\s*\(")
_BOUNDS = re.compile(r"__launch_bounds__\([^)]*\)")


def function_ranges(path):
    """[(first line, last line, name)] of the top-level functions of a source file."""
    out = []
    try:
        lines = open(path).read().splitlines()
    except OSError:
        return out
    i = 0
    while i < len(lines):
        head = _BOUNDS.sub("", lines[i])
        m = _FN_START.match(head)
        if m and not lines[i].rstrip().endswith(";"):
            j = i
            # a one-line body ends on its own line, any other at the next "}" in column 0
            if not lines[i].rstrip().endswith("}"):
                while j < len(lines) and lines[j] != "}":
                    j += 1
            out.append((i + 1, j + 1, m.group(1)))
            i = j
        i += 1
    return out


class Regions:
    def __init__(self):
        self.ranges = {}

    def function(self, path, line):
        if path not in self.ranges:
            self.ranges[path] = function_ranges(path)
        for a, b, name in self.ranges[path]:
            if a <= line <= b:
                return name
        return None

    def region(self, chain, sub):
        if sub:
            return "out-of-line " + sub
        if not chain:
            return "(no line info)"
        path, line = chain[0]
        if not path.startswith(_build.CSRC):
            return "CUDA headers (intrinsics, math)"
        if os.path.basename(path) == "pvq_math.cuh":
            return "pvq_math.cuh, inlined"
        return self.function(path, line) or os.path.basename(path)


def footprint(kernel_filter=None):
    with tempfile.TemporaryDirectory() as tmp:
        cubin, log = compile_cubin(tmp)
        ptx = parse_ptxas(log)
        code = disassemble(cubin)
    rows = []
    for mangled, instrs in code.items():
        name = pretty(mangled)
        if not name.startswith(PVQ_KERNELS):
            continue
        row = {"kernel": name, "mangled": mangled, "sass_bytes": 16 * len(instrs)}
        row.update(ptx.get(mangled, {}))
        for op in COUNTED:
            row[op] = sum(1 for o, _, _ in instrs if o == op)
        rows.append(row)
    rows.sort(key=lambda r: -r["sass_bytes"])
    detail_name = kernel_filter or "k_pvq_persist<true>"
    detail = None
    for mangled, instrs in code.items():
        if pretty(mangled) == detail_name:
            reg = Regions()
            by = {}
            for _, chain, sub in instrs:
                k = reg.region(chain, sub)
                by[k] = by.get(k, 0) + 16
            detail = {"kernel": detail_name, "regions": dict(sorted(by.items(), key=lambda kv: -kv[1]))}
    return rows, detail


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--kernel", help="kernel whose bytes are split by region (default k_pvq_persist<true>)")
    ap.add_argument("--json", action="store_true", help="print one JSON object instead of tables")
    a = ap.parse_args()
    rows, detail = footprint(a.kernel)
    if a.json:
        print(json.dumps({"kernels": rows, "regions": detail}))
        return
    cols = ["sass_bytes", "regs", "stack", "spill_st", "spill_ld"] + list(COUNTED)
    w = max(len(r["kernel"]) for r in rows)
    print("%-*s " % (w, "kernel") + " ".join("%10s" % c for c in cols))
    for r in rows:
        print("%-*s " % (w, r["kernel"]) + " ".join("%10s" % r.get(c, "?") for c in cols))
    if detail:
        print("\n%s: bytes by source region" % detail["kernel"])
        for k, v in detail["regions"].items():
            print("  %-56s %8d" % (k, v))


if __name__ == "__main__":
    main()
