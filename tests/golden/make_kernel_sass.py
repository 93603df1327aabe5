"""Writes tests/golden/kernel_sass.json: per kernel of csrc/kernels.cu, the sha256 of its sm_90a SASS (cuobjdump -sass of
the object build() leaves in csrc/build/kernels.cu.o) and its `-Xptxas -v` resource line.  The probes that only
orchestrate existing kernels (the whole-HBM scan) keep these fixed; tests/test_hbm_scan_abi.py compares a fresh build
with them.

    python tests/golden/make_kernel_sass.py [kernels.cu.o]
"""
import hashlib
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
CSRC = os.path.join(ROOT, "composable-resource-operator_b200", "csrc")
OBJ = os.path.join(CSRC, "build", "kernels.cu.o")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "kernel_sass.json")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC"]


def tool(name):
    return shutil.which(name) or os.path.join("/usr/local/cuda/bin", name)


def sass_digests(obj):
    """{mangled kernel name: sha256 of its SASS lines, whitespace-normalised}"""
    text = subprocess.check_output([tool("cuobjdump"), "-sass", obj], text=True)
    out, name, body = {}, None, []
    for ln in text.splitlines() + ["Function : <end>"]:
        m = re.match(r"\s*Function : (\S+)", ln)
        if m:
            if name:
                out[name] = hashlib.sha256("\n".join(body).encode()).hexdigest()
            name, body = m.group(1), []
        elif name and ln.strip():
            body.append(" ".join(ln.split()))
    out.pop("<end>", None)
    return out


def ptxas_lines():
    """{mangled kernel name: ptxas 'Used ...' line} of a fresh -Xptxas -v compile of kernels.cu"""
    with tempfile.TemporaryDirectory() as d:
        r = subprocess.run([tool("nvcc")] + FLAGS + ["-Xptxas", "-v", "-c", os.path.join(CSRC, "kernels.cu"), "-o",
                                                     os.path.join(d, "k.o")], capture_output=True, text=True, check=True)
    out, name = {}, None
    for ln in (r.stdout + r.stderr).splitlines():
        m = re.search(r"Compiling entry function '(\S+)' for 'sm_90a'", ln)
        if m:
            name = m.group(1)
        elif name and "Used" in ln:
            out[name] = ln.split("ptxas info    :", 1)[-1].strip()
            name = None
    return out


if __name__ == "__main__":
    obj = sys.argv[1] if len(sys.argv) > 1 else OBJ
    json.dump({"sass_sha256": sass_digests(obj), "ptxas": ptxas_lines()}, open(OUT, "w"), indent=1, sort_keys=True)
    print("wrote", OUT)
