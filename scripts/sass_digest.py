#!/usr/bin/env python
"""Per-kernel resource and SASS digest of a CUDA object, library or cubin (cuobjdump; no GPU needed).

    python scripts/sass_digest.py OBJ           one line per function: registers, stack frame, local-memory store / load
                                                 bytes (STL / LDL: ptxas' spill stores and loads), instruction count and
                                                 a hash of the opcode stream (opcodes with modifiers, no operands)
    python scripts/sass_digest.py OBJ_A OBJ_B   the same for both, then only what differs, and a one-line summary

Two builds whose kernels print the same digest run the same instruction stream apart from register numbers, constants and
addresses; a reordering or a changed instruction changes the hash."""
import hashlib
import os
import re
import shutil
import subprocess
import sys

_INSN = re.compile(r"^\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P[T0-9]+\s+)?([A-Z][A-Z0-9_.]*)[^;]*;")
_RES = re.compile(r"REG:(\d+) STACK:(\d+)")
_LOCAL = re.compile(r"^(STL|LDL)\b")
_WIDTH = {"U8": 1, "S8": 1, "U16": 2, "S16": 2, "64": 8, "128": 16}   # modifier -> bytes; none of them: 4


def _tool(name):
    for c in (os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", name), shutil.which(name)):
        if c and os.path.exists(c):
            return c
    sys.exit(f"sass_digest: {name} not found (set CUDA_HOME)")


def _run(*args):
    return subprocess.run(args, check=True, capture_output=True, text=True).stdout


def _demangle(names):
    try:
        out = subprocess.run([_tool("cu++filt")], input="\n".join(names), capture_output=True, text=True, check=True).stdout
        pretty = out.splitlines()
    except (subprocess.CalledProcessError, SystemExit):
        return dict(zip(names, names))
    # drop the return type, the parameter list and the casts of the template arguments, which name the instantiation
    short = [re.sub(r"\((?:int|bool)\)", "", re.sub(r"^void |\([^()]*\)$", "", p)) for p in pretty]
    return dict(zip(names, short)) if len(short) == len(names) else dict(zip(names, names))


def digest(path):
    """{mangled name: dict(regs, stack, stl, ldl, insns, hash)} for every function of the object."""
    cuobjdump = _tool("cuobjdump")
    funcs = {}
    name = None
    for line in _run(cuobjdump, "-res-usage", path).splitlines():
        if line.strip().startswith("Function "):
            name = line.strip()[len("Function "):].rstrip(":")
        elif name and (m := _RES.search(line)):
            funcs[name] = {"regs": int(m[1]), "stack": int(m[2]), "stl": 0, "ldl": 0, "insns": 0, "ops": []}
            name = None
    name = None
    for line in _run(cuobjdump, "-sass", path).splitlines():
        s = line.strip()
        if s.startswith("Function : "):
            name = s[len("Function : "):]
            funcs.setdefault(name, {"regs": -1, "stack": -1, "stl": 0, "ldl": 0, "insns": 0, "ops": []})
            continue
        m = _INSN.match(line)
        if not (name and m):
            continue
        op = m[1]
        f = funcs[name]
        f["insns"] += 1
        f["ops"].append(op)
        if (lm := _LOCAL.match(op)):
            widths = [_WIDTH[mod] for mod in op.split(".")[1:] if mod in _WIDTH]   # e.g. LDL.LU.64: the last width given
            f[lm[1].lower()] += widths[-1] if widths else 4
    for f in funcs.values():
        f["hash"] = hashlib.sha256("\n".join(f.pop("ops")).encode()).hexdigest()[:12]
    return funcs


def _row(name, f):
    return (f"{f['regs']:4d} {f['stack']:5d} {f['stl']:4d} {f['ldl']:4d} {f['insns']:7d}  {f['hash']}  {name}")


HEADER = "regs stack  STL  LDL   insns  opcodes       function"


def main(argv):
    if len(argv) not in (1, 2):
        sys.exit(__doc__)
    digs = [digest(p) for p in argv]
    names = sorted(set().union(*digs))
    pretty = _demangle(names)
    for path, d in zip(argv, digs):
        print(f"== {path}")
        print(HEADER)
        for n in sorted(d, key=lambda n: pretty[n]):
            print(_row(pretty[n], d[n]))
    if len(digs) == 1:
        return 0
    a, b = digs
    print(f"== differences ({argv[0]} -> {argv[1]})")
    same = 0
    for n in sorted(names, key=lambda n: pretty[n]):
        if n not in a or n not in b:
            print(f"only in {'B' if n not in a else 'A'}: {pretty[n]}")
            continue
        fa, fb = a[n], b[n]
        if all(fa[k] == fb[k] for k in ("regs", "stack", "stl", "ldl", "insns", "hash")):
            same += 1
            continue
        print(f"regs {fa['regs']}->{fb['regs']} stack {fa['stack']}->{fb['stack']} STL {fa['stl']}->{fb['stl']} "
              f"LDL {fa['ldl']}->{fb['ldl']} insns {fa['insns']}->{fb['insns']} ({fb['insns'] - fa['insns']:+d})"
              f"{'' if fa['hash'] != fb['hash'] else ' same opcodes'}  {pretty[n]}")
    print(f"{same} of {len(names)} functions identical")
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
