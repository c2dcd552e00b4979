"""Builds libqrl_b200_emu.so: the library's OWN sources (qradiolink_b200/csrc/*.cu, *.cuh) compiled for host threads.

TEST INFRASTRUCTURE ONLY (tests/test_emulated_library.py): lets the CPU tier drive the real host code of qrl_b200.cu -- handle
creation, buffer sizing, launch geometry, slice pipelining, port plumbing -- and the real kernel source through the real C ABI in a
container that has no GPU.  It is not a fallback: the package never looks for it, it is built into a temporary directory by the
test that uses it, and it is orders of magnitude slower than anything useful (one OS thread per CUDA thread).

What the rewrite does to the sources (nothing else is touched):
  * `kernel<<<grid, block, smem, stream>>>(args);`  ->  `emu::launch(dim3(grid), dim3(block), smem, [&] { kernel(args); });`
  * `extern __shared__ T name[];`                   ->  `EMU_DYN_SMEM(T, name);`
  * qrl_tma.cuh (inline PTX: mbarrier, cp.async.bulk, shared-memory loads by address) -> tools/emu/qrl_tma_emu.hpp
  * the other inline-PTX spots of qrl_kernels.cuh: `set.ge.f32.f32` (qrl_ge1), `setp.ge.f32` + `selp.f32` (qrl_sel_ge),
    `set.ge.u32.f32` (qrl_ge_mask) and one `cp.async.bulk.wait_group.read 1`
"""
import os
import re
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
CSRC = os.path.join(ROOT, "qradiolink_b200", "csrc")


def _match(src, i, open_ch, close_ch):
    depth = 0
    while True:
        ch = src[i]
        if ch == open_ch:
            depth += 1
        elif ch == close_ch:
            depth -= 1
            if depth == 0:
                return i
        i += 1


def _split_top(s):
    parts, depth, cur = [], 0, ""
    for ch in s:
        if ch in "([{":
            depth += 1
        elif ch in ")]}":
            depth -= 1
        if ch == "," and depth == 0:
            parts.append(cur.strip()); cur = ""
        else:
            cur += ch
    parts.append(cur.strip())
    return parts


def rewrite_launches(src):
    out, i, n = [], 0, 0
    while True:
        j = src.find("<<<", i)
        if j < 0:
            out.append(src[i:])
            return "".join(out), n
        k = j
        while src[k - 1].isspace():
            k -= 1
        if src[k - 1] == ">":                                   # template arguments of the kernel
            depth, m = 0, k - 1
            while True:
                if src[m] == ">":
                    depth += 1
                elif src[m] == "<":
                    depth -= 1
                    if depth == 0:
                        break
                m -= 1
            k = m
        m = k
        while m > 0 and (src[m - 1].isalnum() or src[m - 1] in "_:"):
            m -= 1
        kern = src[m:j].strip()
        p, depth = j + 3, 0
        while not (depth == 0 and src.startswith(">>>", p)):
            if src[p] in "([{":
                depth += 1
            elif src[p] in ")]}":
                depth -= 1
            p += 1
        cfg = _split_top(src[j + 3:p])
        q = p + 3
        while src[q].isspace():
            q += 1
        assert src[q] == "(", src[j - 80:q + 20]
        r = _match(src, q, "(", ")")
        args = src[q + 1:r]
        grid, block = cfg[0], cfg[1]
        smem = cfg[2] if len(cfg) > 2 else "0"
        out.append(src[i:m])
        out.append("emu::launch(dim3(%s), dim3(%s), %s, [&] { %s(%s); })" % (grid, block, smem, kern, args))
        i = r + 1
        n += 1


def rewrite(src):
    src, n = rewrite_launches(src)
    src = re.sub(r"extern\s+__shared__\s+(?:__align__\(\d+\)\s+)?([\w ]+?)\s+(\w+)\[\];", r"EMU_DYN_SMEM(\1, \2);", src)
    # inline PTX outside qrl_tma.cuh
    src = re.sub(r'asm volatile\("cp\.async\.bulk\.wait_group\.read 1;" ::: "memory"\);', "/* cp.async.bulk.wait_group.read 1 */;", src)
    src = re.sub(r"__device__ __forceinline__ \w+ (qrl_ge1|qrl_sel_ge|qrl_ge_mask)\([^)]*\)[^{]*\{.*?\n\}\n", r"/* \1: tools/emu/qrl_tma_emu.hpp */\n", src, flags=re.S)
    assert "asm" not in re.sub(r"//[^\n]*", "", src).replace("__restrict__", ""), "inline asm left in a rewritten source"
    return src, n


def build(out_dir):
    os.makedirs(out_dir, exist_ok=True)
    total = 0
    for name in os.listdir(CSRC):
        if not name.endswith((".cu", ".cuh", ".hpp")) or name == "qrl_tma.cuh":
            continue
        text = open(os.path.join(CSRC, name)).read()
        if name.endswith((".cu", ".cuh")):
            text, n = rewrite(text)
            total += n
        text = text.replace('#include "../../include/qrl_b200.h"', '#include "%s"' % os.path.join(ROOT, "include", "qrl_b200.h"))
        open(os.path.join(out_dir, name.replace(".cu", ".cpp") if name.endswith(".cu") else name), "w").write(text)
    open(os.path.join(out_dir, "qrl_tma.cuh"), "w").write('#pragma once\n#include <cuda_runtime.h>   // the fake one: pulls in qrl_tma_emu.hpp\n')
    lib = os.path.join(out_dir, "libqrl_b200_emu.so")
    srcs = [os.path.join(out_dir, f) for f in ("qrl_b200.cpp", "qrl_pfb.cpp", "qrl_deframer.cpp", "qrl_spectrum.cpp", "qrl_m17.cpp", "qrl_dmr.cpp")]
    cmd = ["g++", "-std=c++20", "-O" + os.environ.get("QRL_EMU_OPT", "1"), "-ffp-contract=off", "-fno-fast-math", "-pthread", "-fPIC", "-shared", "-Wno-unknown-pragmas",
           "-I", os.path.join(HERE, "fake_cuda"), "-I", HERE, "-I", out_dir, "-o", lib] + srcs
    if os.environ.get("QRL_EMU_ASAN"):      # AddressSanitizer build (CPU memcheck): LD_PRELOAD=$(gcc -print-file-name=libasan.so), ASAN_OPTIONS=detect_leaks=0
        cmd[1:1] = ["-fsanitize=address", "-g"]
    if os.environ.get("QRL_EMU_TSAN"):      # ThreadSanitizer build: load it with LD_PRELOAD=$(gcc -print-file-name=libtsan.so)
        cmd[1:1] = ["-fsanitize=thread", "-g"]
    subprocess.check_call(cmd)
    return lib, total


if __name__ == "__main__":
    lib, n = build(sys.argv[1] if len(sys.argv) > 1 else "/tmp/qrl_emu_build")
    print(lib, "launch sites rewritten:", n)
