"""Pulls named definitions (kernels, device functions, structs, enums, device tables) out of a .cuh as text, each behind the Ring type
and the device functions it calls, rewritten for tools/emu/cuda_emu.hpp: `extern __shared__ T name[];` -> EMU_DYN_SMEM(T, name).  Used by tests/test_kernel_emulation.py."""
import os
import re


def _block_end(src, i):
    depth = 0
    while i < len(src):
        ch = src[i]
        if ch == "{":
            depth += 1
        elif ch == "}":
            depth -= 1
            if depth == 0:
                return i + 1
        i += 1
    raise ValueError("unbalanced braces")


_HERE = os.path.dirname(os.path.abspath(__file__))
_STAND_INS = "".join(open(os.path.join(_HERE, f)).read() for f in ("cuda_emu.hpp", "qrl_tma_emu.hpp"))


def _definition(src, name):
    """The text of the definition of `name` in src, or None."""
    m = (re.search(r"^(?:template\s*<[^\n]*>\s*\n)?(?:__host__\s+)?(?:__global__|__device__)[^;{]*?\b%s\s*\(" % re.escape(name), src, re.M | re.S)
         or re.search(r"^(?:template\s*<[^\n]*>\s*\n)?(?:struct|enum)\s+%s\b[^;{]*\{" % re.escape(name), src, re.M)
         or re.search(r"^enum\s*\{[^}]*\b%s\b" % re.escape(name), src, re.M))
    if m is None:
        m = re.search(r"^(?:__device__|constexpr)[^;\n]*\b%s\b[^;\n]*;" % re.escape(name), src, re.M)       # device table / constant
        return m.group(0) if m else None
    text = src[m.start():_block_end(src, src.index("{", m.start()))]
    if re.match(r"(?:template\s*<[^\n]*>\s*\n)?(?:struct|enum)\b", text.lstrip()):
        text += ";"
    return text


def _dependencies(src, text):
    """What a definition needs ahead of it that the caller may not name: the Ring type of the kernel signatures, and the __device__
    functions it calls that the host-thread stand-ins (cuda_emu.hpp, qrl_tma_emu.hpp) do not provide."""
    deps = ["Ring"] if re.search(r"\bRing\s*<", text) else []
    for name in dict.fromkeys(re.findall(r"\b([A-Za-z]\w*)\s*(?:<[^;(){}]*>)?\s*\(", text)):
        if re.search(r"\b%s\b" % re.escape(name), _STAND_INS):
            continue                                    # the host-thread stand-in replaces the device version
        if re.search(r"^(?:template\s*<[^\n]*>\s*\n)?(?:__host__\s+)?__device__[^;{(]*?\b%s\s*\(" % re.escape(name), src, re.M | re.S):
            deps.append(name)
    return deps


def extract(src, names):
    out, done = [], set()

    def add(name, required):
        if name in done:
            return
        text = _definition(src, name)
        if text is None:
            if required:
                raise KeyError(name)
            return
        done.add(name)
        for dep in _dependencies(src, text):
            add(dep, False)
        out.append(text)

    for name in names:
        add(name, True)
    body = "#ifndef SSP\n#define SSP(...)      /* profiling build only (qrl_kernels.cuh, -DQRL_SS_PROF) */\n#endif\n\n" + "\n\n".join(out)
    body = re.sub(r"extern\s+__shared__\s+(?:__align__\(\d+\)\s+)?([\w ]+?)\s+(\w+)\[\];", r"EMU_DYN_SMEM(\1, \2);", body)
    return body
