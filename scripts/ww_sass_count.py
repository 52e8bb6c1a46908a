"""Static instruction budget of Waterworld's rollout kernels (no GPU needed).

    python scripts/ww_sass_count.py [OBJ_OR_LIB] [--kernel NAME ...] [--all]

Runs `cuobjdump -sass` on a built object or library (default: madrl_b200/build/waterworld.o, which
`python -m madrl_b200.build` leaves behind) and prints, for each named ww_kernel instantiation, the
instruction counts of two loops, with the SHFL, STS and branch (BRA) instructions among them:
  * the per-pursuer loop: the shortest loop (backward branch) that holds an STS, i.e. the one that stages
    a pursuer's feature rows;
  * the step loop: the shortest loop around it that holds a global load (the next step's action prefetch).
Loops nested in these (the candidate scans) are counted as part of them.  Names are the template arguments
after `ww_kernel<float, float, `: `1,1,30,false,0,false,true` is the C2 writer-warp kernel, `1,1,30,false,0,false,false`
the one-warp C2 kernel; `--all` prints every instantiation.
"""
import argparse
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEFAULT_OBJ = os.path.join(ROOT, "madrl_b200", "build", "waterworld.o")
DEFAULT_KERNELS = ["1,1,30,false,0,false,true", "1,1,30,false,0,false,false"]

_INS = re.compile(r"^\s+/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;")
_FUNC = re.compile(r"Function : (\S+)")
# _ZN5madrl9ww_kernelI ff Li1E Li1E Li30E Lb0E Li0E Lb0E Lb1E EEvNS_8WWParams...
_MANGLED = re.compile(r"_ZN5madrl9ww_kernelI(ff|fd|dd|ft)((?:L[ib]-?\d+E)+)EEv")
_REAL = {"f": "float", "d": "double", "t": "uint16_t"}


def demangle(sym):
    """`_ZN5madrl9ww_kernelIffLi1E...` -> ('float,float', '1,1,30,false,0,false,true'), else None."""
    m = _MANGLED.match(sym)
    if not m:
        return None
    types = ",".join(_REAL[c] for c in m.group(1))
    args = []
    for kind, v in re.findall(r"L([ib])(-?\d+)E", m.group(2)):
        args.append(("true" if v == "1" else "false") if kind == "b" else v)
    return types, ",".join(args)


def functions(path):
    """{symbol: [(address, instruction text)]} of every kernel in the cuobjdump -sass listing of `path`."""
    out = subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True, check=True).stdout
    funcs, cur = {}, None
    for line in out.splitlines():
        f = _FUNC.search(line)
        if f:
            cur = funcs.setdefault(f.group(1), [])
            continue
        m = _INS.match(line)
        if m and cur is not None:
            cur.append((int(m.group(1), 16), m.group(2)))
    return funcs


def opcode(text):
    """The opcode of one SASS instruction, without its predicate guard and modifiers."""
    t = re.sub(r"^@!?U?P[T0-9]+\s+", "", text)
    return t.split()[0].split(".")[0] if t else ""


def loops(ins):
    """Every loop as (first, last) instruction index: the target and the source of a backward branch."""
    addr = {a: i for i, (a, _) in enumerate(ins)}
    out = []
    for i, (a, t) in enumerate(ins):
        if opcode(t) != "BRA":
            continue
        m = re.search(r"(0x[0-9a-f]+)\s*$", t)
        if m and int(m.group(1), 16) <= a and int(m.group(1), 16) in addr:
            out.append((addr[int(m.group(1), 16)], i))
    return out


def stats(ins, lo, hi):
    ops = [opcode(t) for _, t in ins[lo:hi + 1]]
    return {"instructions": len(ops), "SHFL": ops.count("SHFL"), "STS": ops.count("STS"), "BRA": ops.count("BRA")}


def budget(ins):
    """{'pursuer loop': stats, 'step loop': stats} of one kernel (a loop that is not found is left out)."""
    ls = loops(ins)
    has = lambda lo, hi, op: any(opcode(t) == op for _, t in ins[lo:hi + 1])
    pursuer = min((l for l in ls if has(*l, "STS")), key=lambda l: l[1] - l[0], default=None)
    if pursuer is None:
        return {}
    res = {"pursuer loop": stats(ins, *pursuer)}
    around = [l for l in ls if l[0] <= pursuer[0] and l[1] >= pursuer[1] and l != pursuer and has(*l, "LDG")]
    if around:
        res["step loop"] = stats(ins, *min(around, key=lambda l: l[1] - l[0]))
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("path", nargs="?", default=DEFAULT_OBJ, help="object or shared library with the ww kernels")
    ap.add_argument("--kernel", action="append", default=[], metavar="ARGS",
                    help="template arguments after the two types, e.g. 1,1,30,false,0,false,true (repeatable)")
    ap.add_argument("--all", action="store_true", help="every ww_kernel instantiation")
    a = ap.parse_args()
    if not os.path.exists(a.path):
        raise SystemExit("%s does not exist (build the library first: python -m madrl_b200.build)" % a.path)
    want = a.kernel or DEFAULT_KERNELS
    found = 0
    for sym, ins in functions(a.path).items():
        d = demangle(sym)
        if d is None or not (a.all or (d[0] == "float,float" and d[1] in want)):
            continue
        found += 1
        print("ww_kernel<%s,%s>  (%d instructions)" % (d[0], d[1], len(ins)))
        for name, s in budget(ins).items():
            print("  %-12s %4d instructions  SHFL %3d  STS %3d  BRA %3d"
                  % (name, s["instructions"], s["SHFL"], s["STS"], s["BRA"]))
    if not found:
        sys.exit("no matching ww_kernel instantiation in %s" % a.path)


if __name__ == "__main__":
    main()
