"""Development aid: are the kernels of two builds the same machine code?  Compiles the raster, spectrum, chain and export kernels of
a base git revision and of the working tree for sm_90a and compares the SASS of every kernel instruction by instruction,
ignoring constant-bank parameter offsets (they move when glava_b200_params grows at its end).  No GPU needed.

    python tools/sass_diff.py <base-rev>
"""
import collections
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "--fmad=false",
         "-Xcompiler", "-fPIC,-ffp-contract=off", "--expt-relaxed-constexpr", "-c"]


def sass(obj):
    out = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
    fn, d = None, collections.OrderedDict()
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            fn = m.group(1); d[fn] = []
            continue
        m = re.match(r"\s+/\*[0-9a-f]+\*/\s+(.*?);", line)
        if m and fn:
            d[fn].append(re.sub(r"c\[0x0\]\[0x[0-9a-f]+\]", "c[PARAM]", m.group(1)))
    return d


def main(base):
    with tempfile.TemporaryDirectory() as tmp:
        wt = os.path.join(tmp, "base")
        subprocess.run(["git", "worktree", "add", "-q", wt, base], cwd=ROOT, check=True)
        try:
            for src in ("raster_kernels.cu", "spectrum_kernels.cu", "chain_kernels.cu", "export_kernels.cu"):
                objs = []
                for tree, tag in ((wt, "base"), (ROOT, "new")):
                    obj = os.path.join(tmp, tag + "_" + src + ".o")
                    subprocess.run(["nvcc"] + FLAGS + ["-o", obj, src], cwd=os.path.join(tree, "glava_b200", "csrc"), check=True,
                                   capture_output=True)
                    objs.append(sass(obj))
                a, b = objs
                for k in b:
                    name = subprocess.run(["c++filt", k], capture_output=True, text=True).stdout.strip().split("(")[0]
                    if k not in a:
                        print(f"{name:48s} new kernel ({len(b[k])} instructions)")
                    else:
                        print(f"{name:48s} base {len(a[k]):5d}  new {len(b[k]):5d}  {'identical' if a[k] == b[k] else 'DIFFERENT'}")
        finally:
            subprocess.run(["git", "worktree", "remove", "--force", wt], cwd=ROOT)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "HEAD")
