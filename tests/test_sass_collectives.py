"""The frontier kernels keep every warp collective converged: in each build of frontier_pack_kernel and frontier_kernel, the
mask of every WARPSYNC.COLLECTIVE (the divergent fallback ptxas puts behind each REDUX / VOTE / SHFL) must be the constant
full mask.  A __reduce_*_sync over a per-run sub-warp mask compiles to a fallback whose mask is a register holding that mask,
entered on every trip once per run; the segmented butterflies in kernel_common.cuh replace it.

The mask's source is found by walking back from the WARPSYNC.COLLECTIVE through the straight-line code before it to the
instruction that wrote the mask register, following register copies.  A walk that meets an unconditional branch, a predicated
or unknown write, or the start of the kernel before it finds a constant fails the test: an unresolved mask is not a pass.

CPU only: reads the SASS of the built library, or of fresh sm_90a cubins when the library has not been built."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "bobrapet_b200", "csrc")
LIB = os.path.join(ROOT, "bobrapet_b200", "lib", "libbobrafrontier.so")
CUDA_BIN = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin")
KERNELS = ("frontier_pack_kernel", "frontier_kernel")


def _tool(name):
    return shutil.which(name) or (os.path.join(CUDA_BIN, name) if os.path.exists(os.path.join(CUDA_BIN, name)) else None)


def _sass(tmp_path_factory):
    cuobjdump = _tool("cuobjdump")
    if cuobjdump is None:
        pytest.skip("cuobjdump not found")
    if os.path.exists(LIB):
        return subprocess.run([cuobjdump, "-sass", LIB], capture_output=True, text=True, check=True).stdout
    nvcc = _tool("nvcc")
    if nvcc is None:
        pytest.skip("neither a built library nor nvcc")
    out = tmp_path_factory.mktemp("sass")
    text = []
    for src in ("frontier_pack.cu", "frontier_kernel.cu"):
        cubin = str(out / (src + ".cubin"))
        subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-cubin", "-o", cubin,
                        os.path.join(CSRC, src)], check=True, capture_output=True)
        text.append(subprocess.run([cuobjdump, "-sass", cubin], capture_output=True, text=True, check=True).stdout)
    return "\n".join(text)


def _functions(sass):
    """{mangled name: [instruction text, in address order]} of the frontier kernels"""
    funcs, cur = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            cur = name if any(re.match(r"_ZN2bf\d+%s[IE]" % k, name) for k in KERNELS) else None
            if cur:
                funcs[cur] = []
            continue
        m = re.match(r"\s+/\*[0-9a-f]+\*/\s+(.*?)\s*;", line)
        if cur and m:
            funcs[cur].append(m.group(1))
    return funcs


def _mask_source(ins, i, reg):
    """the constant written to `reg` on the straight-line path into instruction i, or None (unresolved)"""
    for j in range(i - 1, -1, -1):
        t = ins[j]
        if re.match(r"(BRA|JMP|EXIT|RET)\b", t):   # unconditional: the path into i does not come from here
            return None
        m = re.match(r"(@!?U?P\w+\s+)?([A-Z0-9_.]+)\s*(.*)", t)
        if m is None:
            return None
        pred, op, args = m.group(1), m.group(2), m.group(3).split(", ")
        if op.startswith(("WARPSYNC", "ST", "RED", "BSSY", "BSYNC")):
            continue
        if op.startswith("SHFL") and len(args) > 1 and args[1] == reg:   # SHFL's second destination
            return None
        d = re.fullmatch(r"R(\d+)", args[0])
        width = 4 if ".128" in op else (2 if (".64" in op or "WIDE" in op) else 1)
        if d is None or not int(d.group(1)) <= int(reg[1:]) < int(d.group(1)) + width:
            continue
        if width > 1 or args[0] != reg:   # part of a wide write
            return None
        if pred:
            return None
        if op == "IMAD.MOV.U32" and args[1:3] == ["RZ", "RZ"]:
            src = args[3]
        elif op == "MOV":
            src = args[1]
        else:
            return None
        if re.fullmatch(r"R\d+", src):
            return _mask_source(ins, j, src)
        return src
    return None


def test_collective_masks_are_full(tmp_path_factory):
    funcs = _functions(_sass(tmp_path_factory))
    for k in KERNELS:
        assert any(re.match(r"_ZN2bf\d+%s[IE]" % k, f) for f in funcs), "no %s build in the SASS" % k
    bad = []
    for name, ins in funcs.items():
        for i, t in enumerate(ins):
            m = re.match(r"WARPSYNC\.COLLECTIVE (\w+),", t)
            if not m:
                continue
            src = _mask_source(ins, i, m.group(1))
            if src not in ("-0x1", "0xffffffff"):
                bad.append("%s: %s before %s (mask: %s)" % (name, t, ins[i + 1], src or "unresolved"))
    assert not bad, "collectives with a per-lane mask:\n" + "\n".join(bad)
