#!/usr/bin/env python
"""Compare the SASS of two builds of libnastar_b200.so kernel by kernel.

    python tools/sass_diff.py old.so new.so [-v]

Runs `cuobjdump -sass` on both libraries and pairs their functions by demangled name.  The search engines' former
argument structs (W32Args, W64Args, GenArgs) are read as SearchArgs, and heur32_init_kernel<k> / heur64_init_kernel<k>
as heur_init_kernel<32, k> / heur_init_kernel<64, k>, so that a build from before the shared engine scaffold pairs
with one after it.  Each kernel is reported as
  identical          the same instructions and encodings;
  param-offsets      the same instructions once kernel-parameter constant-bank offsets (c[0x0][0x210] and up on
                     sm_90) are masked: a parameter moved inside the argument struct, nothing else changed;
  different          anything else (-v prints the first differing instructions);
  only-old/only-new  present in one library only.
Exits 1 if any kernel is different or present in one library only, else 0.
"""
import argparse
import collections
import difflib
import os
import re
import shutil
import subprocess
import sys

PARAM_BASE = 0x210   # first kernel-parameter byte in constant bank 0 on sm_90
_FUNC = re.compile(r"^\s+Function : (\S+)")
_INSN = re.compile(r"^\s+/\*[0-9a-f]{4,}\*/\s+(.*?;)\s*(/\* 0x[0-9a-f]+ \*/)?\s*$")
_ENC = re.compile(r"^\s+(/\* 0x[0-9a-f]+ \*/)\s*$")
_CBANK = re.compile(r"c\[0x0\]\[0x([0-9a-f]+)\]")
_RENAMES = [(re.compile(r"\bnastar::(?:W32Args|W64Args|GenArgs)\b"), "nastar::SearchArgs"),
            (re.compile(r"\bheur(32|64)_init_kernel<"), r"heur_init_kernel<\1, "),
            (re.compile(r"_GLOBAL__N__\w+"), "(anonymous namespace)")]


def tool(name):
    path = shutil.which(name) or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", name)
    if not os.path.exists(path):
        sys.exit(f"sass_diff: {name} not found (put the CUDA toolkit's bin/ on PATH or set CUDA_HOME)")
    return path


def kernels(lib):
    """{paired name: [(instruction, encoding), ...]} of every function in `lib`'s sm_90a code."""
    out = subprocess.run([tool("cuobjdump"), "-sass", lib], capture_output=True, text=True, check=True).stdout
    funcs, cur = collections.OrderedDict(), None
    for ln in out.splitlines():
        m = _FUNC.match(ln)
        if m:
            cur = funcs.setdefault(m.group(1), [])
            continue
        if cur is None:
            continue
        m = _INSN.match(ln)
        if m:
            cur.append([m.group(1), m.group(2) or ""])
            continue
        m = _ENC.match(ln)
        if m and cur:
            cur[-1][1] += m.group(1)
    mangled = list(funcs)
    demangled = subprocess.run([tool("c++filt")], input="\n".join(mangled), capture_output=True, text=True,
                               check=True).stdout.splitlines()
    named = collections.OrderedDict()
    for m, d in zip(mangled, demangled):
        for pat, rep in _RENAMES:
            d = pat.sub(rep, d)
        if d in named:
            sys.exit(f"sass_diff: {lib}: two functions pair as {d}")
        named[d] = funcs[m]
    return named


def mask_params(ins):
    return _CBANK.sub(lambda m: "c[0x0][PARAM]" if int(m.group(1), 16) >= PARAM_BASE else m.group(0), ins)


def compare(a, b):
    if a == b:
        return "identical"
    if [mask_params(i) for i, _ in a] == [mask_params(i) for i, _ in b]:
        return "param-offsets"
    return "different"


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("old")
    ap.add_argument("new")
    ap.add_argument("-v", "--verbose", action="store_true", help="print the first lines that differ per kernel")
    args = ap.parse_args()
    old, new = kernels(args.old), kernels(args.new)
    counts = collections.Counter()
    for name in list(old) + [n for n in new if n not in old]:
        if name not in new:
            status = "only-old"
        elif name not in old:
            status = "only-new"
        else:
            status = compare(old[name], new[name])
        counts[status] += 1
        print(f"{status:14s} {name}")
        if args.verbose and status == "different":
            diff = difflib.unified_diff([i for i, _ in old[name]], [i for i, _ in new[name]], lineterm="", n=1)
            for ln in list(diff)[2:22]:
                print("    " + ln)
    print("# " + ", ".join(f"{k}: {counts[k]}" for k in ("identical", "param-offsets", "different", "only-old",
                                                          "only-new")))
    return 1 if counts["different"] or counts["only-old"] or counts["only-new"] else 0


if __name__ == "__main__":
    sys.exit(main())
