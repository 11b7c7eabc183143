"""Build check: the kernels a base revision of td_diffusion.cu had compile to the same SASS, instruction for instruction, in the
working tree; and the -Xptxas -v registers and spills of the kernels the working tree adds.

    python tests/debug_tools/sass_identity.py [--base HEAD~1]

Compiles both versions of csrc/td_diffusion.cu to cubins with the library's nvcc flags (no GPU needed), disassembles them
with cuobjdump -sass and compares each base kernel's instructions with the working tree's kernel of the same name.  A
template parameter the tree appends with a default (e.g. SPARSE = false) and trailing pointer parameters the base kernel did
not have are dropped from the tree's names before matching.  Exits 1 when a base kernel is missing or differs.
"""
import argparse
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
PKG = os.path.join(ROOT, "multidiffusion_upscaler_for_automatic1111_b200")
SRC = "multidiffusion_upscaler_for_automatic1111_b200/csrc/td_diffusion.cu"
sys.path.insert(0, PKG)
from build import NVCC_FLAGS  # noqa: E402

NVCC = "/usr/local/cuda/bin/nvcc"
CUOBJDUMP = "/usr/local/cuda/bin/cuobjdump"


def compile_cubin(src, out):
    flags = [f for f in NVCC_FLAGS if f not in ("--shared", "-Xcompiler", "-fPIC,-ffp-contract=off")]
    cmd = [NVCC, *flags, "-Xcompiler", "-ffp-contract=off", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(PKG, "csrc"),
           "-cubin", "-o", out, src]
    res = subprocess.run(cmd, capture_output=True, text=True, check=True)
    return res.stdout + res.stderr


def functions(cubin):
    out, cur = {}, None
    for line in subprocess.run([CUOBJDUMP, "-sass", cubin], capture_output=True, text=True, check=True).stdout.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            out[cur] = []
        elif cur is not None and re.match(r"\s*/\*[0-9a-f]{4}\*/", line):
            out[cur].append(line.strip())
    return out


def demangle(names):
    res = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True).stdout.splitlines()
    return dict(zip(names, res))


SPARSE_KERNELS = ("blend_md_async_kernel", "blend_mod_async_kernel", "blend_grid_generic_kernel")   # SPARSE = false appended


def normalise(name):
    for k in SPARSE_KERNELS:
        if k + "<" in name:
            name = re.sub(k + r"(<[^()]*?), false>", k + r"\1>", name)
            return re.sub(r", int const\*\)$", ")", name)
    return name


def ptxas_info(log):
    """{mangled name: (registers, spill stores, spill loads)}."""
    info, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur:
            info.setdefault(cur, [0, 0, 0])[1:] = [int(m.group(1)), int(m.group(2))]
        m = re.search(r"Used (\d+) registers", line)
        if m and cur:
            info.setdefault(cur, [0, 0, 0])[0] = int(m.group(1))
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", default="HEAD~1", help="git revision of the base td_diffusion.cu")
    args = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        base_src = os.path.join(tmp, "td_diffusion.cu")
        with open(base_src, "w") as f:
            f.write(subprocess.run(["git", "-C", ROOT, "show", f"{args.base}:{SRC}"], capture_output=True, text=True, check=True).stdout)
        compile_cubin(base_src, os.path.join(tmp, "base.cubin"))
        log = compile_cubin(os.path.join(ROOT, SRC), os.path.join(tmp, "tree.cubin"))
        base, tree = functions(os.path.join(tmp, "base.cubin")), functions(os.path.join(tmp, "tree.cubin"))
    db, dt = demangle(list(base)), demangle(list(tree))
    by_name = {normalise(dt[k]): k for k in tree}
    bad = 0
    for k, body in base.items():
        twin = by_name.get(db[k])
        if twin is None or tree[twin] != body:
            bad += 1
            print(("MISSING " if twin is None else "DIFFERS ") + db[k])
    matched = {by_name[db[k]] for k in base if db[k] in by_name}
    print(f"{len(base) - bad} of {len(base)} base kernels identical")
    info = ptxas_info(log)
    for k in sorted(set(tree) - matched, key=lambda n: dt[n]):
        regs, st, ld = info.get(k, (0, 0, 0))
        short = re.sub(r"\(anonymous namespace\)::", "", dt[k]).split("(")[0]
        print(f"new: {short:<70} {regs:3d} registers, spills {st}/{ld} bytes")
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
