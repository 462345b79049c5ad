"""md5 of the SASS instruction stream of every step kernel in libdojo_b200.so (or another build of it).

    python tools/sass_md5.py [LIB]

One line per kernel: md5 of its instructions as `cuobjdump -sass` prints them (text only: addresses and encodings are dropped),
instruction count, demangled name.  Two builds whose untraced kernels print the same md5 run the same machine code; the names are
printed demangled and trailing TRACE = false / SMALL = false / REC = false / FB = false / VJP = false template arguments are dropped, so
that builds before and after the traced, the small-mechanism, the recording-rollout, the closed-loop and the adjoint kernels were added
can be compared line by line (DESIGN.md section 6).
"""
import hashlib
import os
import re
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def kernels(lib):
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    text = subprocess.run([cuobjdump, "-sass", lib], check=True, capture_output=True, text=True).stdout
    out, name, ins = {}, None, []
    for line in text.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            if name:
                out[name] = ins
            name, ins = m.group(1), []
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(.*?)\s*;", line)
        if m and name:
            ins.append(m.group(1))
    if name:
        out[name] = ins
    return out


def demangle(names):
    r = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True, check=True).stdout.split("\n")
    return [re.sub(r"void (.*)\(.*", r"\1", d) for d in r[: len(names)]]


def main():
    lib = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "dojo.jl_b200", "libdojo_b200.so")
    ks = {n: v for n, v in kernels(lib).items() if "dojo_step_kernel" in n}
    for mangled, name in sorted(zip(ks, demangle(list(ks))), key=lambda t: t[1]):
        m = re.match(r"(.*)<(.*)>$", name)
        if m:  # <GRAD, PLAN_SMEM[, TRACE[, SMALL[, REC[, FB[, VJP]]]]]>: defaulted trailing arguments are not printed
            args = m.group(2).split(", ")
            while len(args) > 2 and args[-1] == "false":
                args.pop()
            name = f"{m.group(1)}<{', '.join(args)}>"
        ins = ks[mangled]
        print(f"{hashlib.md5(chr(10).join(ins).encode()).hexdigest()}  {len(ins):6d}  {name}")


if __name__ == "__main__":
    main()
