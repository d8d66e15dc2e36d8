"""TEST INFRASTRUCTURE: builds tests/cuda_emu/_build/libb200z_emu.so -- the UNMODIFIED sources of sharpziplib_b200/csrc compiled
for the CPU on top of cuda_emu.h (fibers as CUDA threads).  Two textual rewrites, nothing else:
  kernel<<<grid, block, smem, stream>>>(args);   ->  EMU_LAUNCH(kernel, grid, block, smem, args);
  extern __shared__ [__align__(n)] uint8_t name[];  ->  uint8_t *name = emu::dyn_smem();
The product never loads this library; tests/cuda_emu/run_emulated.py swaps it in inside the test process."""
import os
import re
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
# B200Z_EMU_CSRC / B200Z_EMU_OUT: build from another copy of the kernel sources (e.g. one with an experimental patch applied)
CSRC = os.environ.get("B200Z_EMU_CSRC", os.path.join(ROOT, "sharpziplib_b200", "csrc"))
OUT = os.environ.get("B200Z_EMU_OUT", os.path.join(HERE, "_build"))


def _split_top(s):
    parts, depth, cur = [], 0, ""
    for ch in s:
        if ch in "([{":
            depth += 1
        elif ch in ")]}":
            depth -= 1
        if ch == "," and depth == 0:
            parts.append(cur.strip())
            cur = ""
        else:
            cur += ch
    parts.append(cur.strip())
    return parts


def rewrite(src):
    out, i = "", 0
    while True:
        j = src.find("<<<", i)
        if j < 0:
            out += src[i:]
            break
        # kernel name (identifier, optionally with template arguments) right in front of <<<
        k = j
        if src[k - 1] == ">":
            depth = 0
            while True:
                k -= 1
                if src[k] == ">":
                    depth += 1
                elif src[k] == "<":
                    depth -= 1
                    if depth == 0:
                        break
        while k > 0 and (src[k - 1].isalnum() or src[k - 1] == "_"):
            k -= 1
        name = src[k:j]
        e = src.index(">>>", j)
        cfg = _split_top(src[j + 3:e])
        assert len(cfg) == 4, cfg
        a0 = src.index("(", e)
        depth, a1 = 0, a0
        while True:
            if src[a1] == "(":
                depth += 1
            elif src[a1] == ")":
                depth -= 1
                if depth == 0:
                    break
            a1 += 1
        args = src[a0 + 1:a1]
        if "," in name:  # template arguments: keep the macro from splitting them
            name = "(" + name + ")"
        out += src[i:k] + "EMU_LAUNCH(%s, %s, %s, %s, %s)" % (name, cfg[0], cfg[1], cfg[2], args)
        i = a1 + 1
    out = re.sub(r"extern\s+__shared__\s+(?:__align__\(\d+\)\s+)?uint8_t\s+(\w+)\[\];", r"uint8_t *\1 = emu::dyn_smem();", out)
    return out


def build(sanitize=False, verbose=False):
    """sanitize: False, True / "ub" (UBSan) or "asan" (AddressSanitizer: cudaMalloc'ed memory is heap memory, so a kernel
    that reads or writes outside its buffers is reported; run python with LD_PRELOAD=libasan and detect_leaks=0)"""
    os.makedirs(os.path.join(OUT, "src"), exist_ok=True)
    so = os.path.join(OUT, "libb200z_emu%s.so" % ("_asan" if sanitize == "asan" else "_san" if sanitize else ""))
    files = sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))
    srcs = [os.path.join(CSRC, f) for f in files]
    deps = srcs + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cuh")] + \
        [os.path.join(HERE, "cuda_emu.h"), os.path.join(HERE, "cuda_emu.cpp"), os.path.abspath(__file__),
         os.path.join(os.path.dirname(os.path.dirname(CSRC)), "include", "b200z.h")]
    if os.path.exists(so) and all(os.path.getmtime(so) >= os.path.getmtime(d) for d in deps):
        return so
    gen = []
    for f in files:
        text = open(os.path.join(CSRC, f)).read()
        dst = os.path.join(OUT, "src", f.replace(".cu", ".cpp"))
        # headers are found next to the original sources
        open(dst, "w").write('#line 1 "%s"\n' % os.path.join(CSRC, f) + rewrite(text))
        gen.append(dst)
    # headers with kernels of their own (dynamic shared memory declarations, launches): rewritten next to the sources
    for f in os.listdir(CSRC):
        if f.endswith(".cuh"):
            text = open(os.path.join(CSRC, f)).read()
            if "extern __shared__" in text or "<<<" in text:
                open(os.path.join(OUT, "src", f), "w").write('#line 1 "%s"\n' % os.path.join(CSRC, f) + rewrite(text))
    # headers that declare dynamic shared memory themselves (experimental kernels #included by a patched source)
    exp = os.path.join(CSRC, "experimental")
    if os.path.isdir(exp):
        os.makedirs(os.path.join(OUT, "src", "experimental"), exist_ok=True)
        for f in os.listdir(exp):
            if f.endswith(".cuh"):
                open(os.path.join(OUT, "src", "experimental", f), "w").write(rewrite(open(os.path.join(exp, f)).read()))
    flags = ["-std=c++17", "-O1", "-g", "-fPIC", "-shared", "-w"] + os.environ.get("B200Z_EMU_CXXFLAGS", "").split() + [ "-I", os.path.join(HERE, "include"),
             "-iquote", os.path.join(OUT, "src"), "-I", CSRC, "-iquote", CSRC]
    if sanitize == "asan":
        flags += ["-fsanitize=address", "-fno-omit-frame-pointer"]
    elif sanitize:
        flags += ["-fsanitize=undefined", "-fno-sanitize-recover=undefined", "-fno-sanitize=alignment"]
    cmd = ["g++"] + flags + ["-o", so] + gen + [os.path.join(HERE, "cuda_emu.cpp")]
    if verbose:
        print(" ".join(cmd))
    subprocess.check_call(cmd)
    return so


if __name__ == "__main__":
    print(build(sanitize="asan" if "--asan" in sys.argv else "--sanitize" in sys.argv, verbose=True))
