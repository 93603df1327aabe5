"""Writes the SASS pins of the kernel translation units: per kernel, the sha256 of its sm_90a SASS (cuobjdump -sass of
the object build() leaves in csrc/build/<source>.o) and its `-Xptxas -v` resource line.

  kernel_sass.json     csrc/kernels.cu: the probes that only orchestrate existing kernels (the whole-HBM scan) keep
                       these fixed; tests/test_hbm_scan_abi.py compares a fresh build with them.
  precision_sass.json  csrc/precision_kernels.cu: tests/test_precision_abi.py compares a fresh build with them.

Kernel names are taken with nvcc's anonymous-namespace tag, which changes with the file, replaced by `_GLOBAL__N_`.

    python tests/golden/make_kernel_sass.py [kernels.cu | precision_kernels.cu] [object]
"""
import hashlib
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
CSRC = os.path.join(ROOT, "composable-resource-operator_b200", "csrc")
PINS = {"kernels.cu": "kernel_sass.json", "precision_kernels.cu": "precision_sass.json"}
OBJ = os.path.join(CSRC, "build", "kernels.cu.o")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC"]


def tool(name):
    return shutil.which(name) or os.path.join("/usr/local/cuda/bin", name)


def obj_of(src):
    return os.path.join(CSRC, "build", src + ".o")


def kernel_name(mangled):
    """mangled with its anonymous-namespace component (<length>_GLOBAL__N__<hash>_<n>_<file>_<hash>) as _GLOBAL__N_"""
    m = re.search(r"(\d+)_GLOBAL__N__", mangled)
    if not m:
        return mangled
    return mangled[:m.start()] + "11_GLOBAL__N_" + mangled[m.end(1) + int(m.group(1)):]


def sass_digests(obj):
    """{mangled kernel name: sha256 of its SASS lines, whitespace-normalised}"""
    text = subprocess.check_output([tool("cuobjdump"), "-sass", obj], text=True)
    out, name, body = {}, None, []
    for ln in text.splitlines() + ["Function : <end>"]:
        m = re.match(r"\s*Function : (\S+)", ln)
        if m:
            if name:
                out[kernel_name(name)] = hashlib.sha256("\n".join(body).encode()).hexdigest()
            name, body = m.group(1), []
        elif name and ln.strip():
            body.append(" ".join(ln.split()))
    out.pop("<end>", None)
    return out


def ptxas_lines(src="kernels.cu"):
    """{mangled kernel name: ptxas 'Used ...' line} of a fresh -Xptxas -v compile of csrc/src"""
    with tempfile.TemporaryDirectory() as d:
        r = subprocess.run([tool("nvcc")] + FLAGS + ["-Xptxas", "-v", "-c", os.path.join(CSRC, src), "-o",
                                                     os.path.join(d, "k.o")], capture_output=True, text=True, check=True)
    out, name = {}, None
    for ln in (r.stdout + r.stderr).splitlines():
        m = re.search(r"Compiling entry function '(\S+)' for 'sm_90a'", ln)
        if m:
            name = kernel_name(m.group(1))
        elif name and "Used" in ln:
            out[name] = ln.split("ptxas info    :", 1)[-1].strip()
            name = None
    return out


if __name__ == "__main__":
    src = sys.argv[1] if len(sys.argv) > 1 else "kernels.cu"
    obj = sys.argv[2] if len(sys.argv) > 2 else obj_of(src)
    out = os.path.join(HERE, PINS[src])
    json.dump({"sass_sha256": sass_digests(obj), "ptxas": ptxas_lines(src)}, open(out, "w"), indent=1, sort_keys=True)
    print("wrote", out)
