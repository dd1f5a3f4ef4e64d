#!/usr/bin/env python3
"""Compare the device code of two builds of the product library, function by function.

    python scripts/compare_device_code.py OLD_TREE NEW_TREE

Each tree is a checkout in which `make -C edlib_b200/csrc` has run.  The script compares
  * the SASS of every kernel (`cuobjdump -sass edlib_b200/lib/libedlib_b200.so`, split at `Function :`), and
  * the ptxas resource lines of every kernel (registers, shared memory, stack, spills) in edlib_b200/lib/ptxas.log,
so the order in which the compiler emitted the functions does not matter.  It exits with 1 and prints the
differences when the device code differs.  Needs no GPU: a host-side change (launch code, dispatch) that leaves
this output identical cannot have changed what the kernels execute.
"""
import difflib
import os
import re
import shutil
import subprocess
import sys


def cuobjdump():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe):
        sys.exit("cuobjdump not found (CUDA toolkit)")
    return exe


def sass_functions(lib):
    out = subprocess.run([cuobjdump(), "-sass", lib], check=True, capture_output=True, text=True).stdout
    funcs, name = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            funcs[name] = []
        elif name is not None:
            funcs[name].append(line.rstrip())
    return funcs


def ptxas_resources(log):
    """{function: [resource lines]} and the number of kernels compiled."""
    res, name, kernels = {}, None, 0
    with open(log) as f:
        for line in f:
            line = line.strip()
            m = re.search(r"Compiling entry function '([^']+)'", line)
            if m:
                kernels += 1
                name = m.group(1)
                continue
            m = re.search(r"Function properties for (\S+)", line)
            if m:
                name = m.group(1)
                continue
            if name and ("bytes stack frame" in line or line.startswith("ptxas info    : Used")):
                res.setdefault(name, []).append(line)
    return res, kernels


def compare(label, old, new):
    bad = 0
    for name in sorted(set(old) | set(new)):
        if name not in new:
            print(f"{label}: {name} only in the old build")
        elif name not in old:
            print(f"{label}: {name} only in the new build")
        elif old[name] != new[name]:
            print(f"{label}: {name} differs")
            sys.stdout.writelines(difflib.unified_diff([l + "\n" for l in old[name]], [l + "\n" for l in new[name]], n=1))
        else:
            continue
        bad += 1
    return bad


def main():
    if len(sys.argv) != 3:
        sys.exit(__doc__)
    lib = lambda tree, f: os.path.join(tree, "edlib_b200", "lib", f)
    old_tree, new_tree = sys.argv[1:]
    old_sass, new_sass = sass_functions(lib(old_tree, "libedlib_b200.so")), sass_functions(lib(new_tree, "libedlib_b200.so"))
    (old_res, old_k), (new_res, new_k) = ptxas_resources(lib(old_tree, "ptxas.log")), ptxas_resources(lib(new_tree, "ptxas.log"))
    bad = compare("sass", old_sass, new_sass) + compare("ptxas", old_res, new_res)
    if old_k != new_k:
        print(f"ptxas: {old_k} kernels compiled in the old build, {new_k} in the new one")
        bad += 1
    print(f"{len(old_sass)} / {len(new_sass)} SASS functions, {old_k} / {new_k} kernels compiled: "
          + ("identical" if bad == 0 else f"{bad} differences"))
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
