"""TEST INFRASTRUCTURE: builds tests/emu/_build/libhorae_emu.so — the product's own sources (horaedb_b200/csrc/*.cu, parquet_meta.cpp,
inspect.cpp) compiled by g++ against tests/emu/cuda_emu.h, so the kernels run on the CPU with every thread as a coroutine.

The sources are used as they are except for what g++ cannot parse:
  * `kernel<<<grid, block, smem, stream>>>(args)`  ->  `EMU_LAUNCH((kernel), grid, block, smem, stream, args)`
  * `extern __shared__ T name[];`                   ->  `EMU_DYN_SMEM(T, name);`
  * inline PTX outside `#ifdef __CUDACC__` (L2 prefetches, `ld.global.cg`) -> nothing / a plain load
  * comm.cu's `dlopen("libnccl.so.2")` -> tests/emu/nccl_emu.cpp (ranks = threads of the test process)
snappy_core.h / zstd_core.h select their host variants by `#ifdef __CUDACC__`, exactly as for tests/emu/snappy_emu.cpp; kernels.h
sets the SM count `kNumSMs` to 4 under HORAE_EMULATED_BUILD.
Nothing in horaedb_b200/ knows this library exists."""
import os
import re
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.normpath(os.path.join(HERE, "..", ".."))
CSRC = os.path.join(ROOT, "horaedb_b200", "csrc")
# HORAE_EMU_DROP_BARRIER=file.cu:N[:warp] builds a MUTANT without the N-th __syncthreads() (or __syncwarp()) of that file, into its own directory: how the
# sensitivity of the emulated runs is measured (a mutant that passes every test under every thread order is a barrier the tests do not need)
MUTANT = os.environ.get("HORAE_EMU_DROP_BARRIER", "")
_TAG = ("_mut_" + MUTANT.replace(".", "_").replace(":", "_")) if MUTANT else ""
BUILD = os.path.join(HERE, "_build", "engine" + _TAG)
OUT = os.path.join(HERE, "_build", "libhorae_emu%s.so" % _TAG)
NCCL_OUT = os.path.join(HERE, "_build", "libnccl_emu.so")
CU = ["engine.cu", "kernels.cu", "fused_scan.cu", "snappy.cu", "zstd.cu", "kway_merge.cu", "radix_agg.cu", "comm.cu", "sst_writer.cu"]
CPP = ["parquet_meta.cpp", "inspect.cpp"]


def _match_back_template(s, i):
    """s[i] == '>' closing a template argument list: index of the matching '<'."""
    depth = 0
    while i >= 0:
        if s[i] == ">":
            depth += 1
        elif s[i] == "<":
            depth -= 1
            if depth == 0:
                return i
        i -= 1
    raise ValueError("unbalanced template arguments before <<<")


def _split_top(s):
    parts, depth, cur = [], 0, []
    for ch in s:
        if ch in "([{":
            depth += 1
        elif ch in ")]}":
            depth -= 1
        if ch == "," and depth == 0:
            parts.append("".join(cur).strip())
            cur = []
        else:
            cur.append(ch)
    parts.append("".join(cur).strip())
    return parts


def rewrite_launches(s):
    out, pos = [], 0
    while True:
        i = s.find("<<<", pos)
        if i < 0:
            out.append(s[pos:])
            return "".join(out)
        # kernel expression: identifier (with namespaces) and optional template arguments, right before <<<
        j = i - 1
        while s[j].isspace():
            j -= 1
        if s[j] == ">":
            j = _match_back_template(s, j) - 1
            while s[j].isspace():
                j -= 1
        k = j
        while k >= 0 and (s[k].isalnum() or s[k] in "_:"):
            k -= 1
        kernel = s[k + 1:i].strip()
        m = re.compile(r">>>\s*\(").search(s, i)
        cfg = _split_top(s[i + 3:m.start()])
        assert 2 <= len(cfg) <= 4, cfg
        cfg += ["0"] * (4 - len(cfg))
        a = m.end()                                  # first char after '('
        depth, e = 1, a
        while depth:
            if s[e] == "(":
                depth += 1
            elif s[e] == ")":
                depth -= 1
            e += 1
        args = s[a:e - 1].strip()
        out.append(s[pos:k + 1])
        out.append("EMU_LAUNCH((%s), %s%s)" % (kernel, ", ".join(cfg), (", " + args) if args else ""))
        pos = e


def transform(text, name=""):
    if MUTANT and MUTANT.split(":")[0] == name:
        parts = MUTANT.split(":")
        n, pos, tok = int(parts[1]), -1, ("__syncwarp();" if len(parts) > 2 and parts[2] == "warp" else "__syncthreads();")
        for _ in range(n + 1):
            pos = text.find(tok, pos + 1)
            if pos < 0:
                raise SystemExit("no such barrier: " + MUTANT)
        text = text[:pos] + "/* dropped */" + " " * (len(tok) - 13) + text[pos + len(tok):]
    text = rewrite_launches(text)
    text = re.sub(r"extern\s+__shared__\s+([\w:]+)\s+(\w+)\s*\[\s*\]\s*;", r"EMU_DYN_SMEM(\1, \2);", text)
    text = re.sub(r'asm volatile\("prefetch\.global\.L2 \[%0\];"[^;]*;', "(void)0;", text)
    text = re.sub(r'asm volatile\("ld\.global\.cg\.u(?:8|16|32|64) %0, \[%1\];" : "=[rl]"\((\w+)\) : "l"\((\w+)\)\);', r"\1 = *\2;", text)
    text = text.replace('"libnccl.so.2", "libnccl.so"', '"%s"' % NCCL_OUT)       # comm.cu binds NCCL with dlopen: the test's stand-in
    return text


def build(force=False):
    os.makedirs(BUILD, exist_ok=True)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cpp", ".h", ".hpp"))]
    deps += [os.path.join(HERE, "cuda_emu.h"), os.path.join(HERE, "engine_emu_glue.cpp"), os.path.join(HERE, "nccl_emu.cpp"), os.path.abspath(__file__), os.path.join(ROOT, "include", "horae_gpu.h")]
    if not force and os.path.exists(OUT) and os.path.getmtime(OUT) >= max(os.path.getmtime(d) for d in deps):
        return OUT
    shim = os.path.join(BUILD, "shim")
    os.makedirs(shim, exist_ok=True)
    with open(os.path.join(shim, "cuda_runtime.h"), "w") as f:
        f.write('#pragma once\n#include "%s"\n' % os.path.join(HERE, "cuda_emu.h"))
    objs, procs = [], []
    flags = ["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-w", "-D__grid_constant__=", "-DHORAE_EMULATED_BUILD", "-I", shim, "-I", CSRC, "-I", os.path.join(ROOT, "include")]
    for name in CU:
        src = os.path.join(BUILD, name.replace(".cu", "_emu.cpp"))
        with open(os.path.join(CSRC, name)) as f:
            text = transform(f.read(), name)
        with open(src, "w") as f:
            f.write('#include "cuda_runtime.h"\n#line 1 "%s"\n' % os.path.join(CSRC, name) + text)
        obj = src[:-4] + ".o"
        procs.append((subprocess.Popen(flags + ["-c", src, "-o", obj]), name))
        objs.append(obj)
    for name in CPP + ["engine_emu_glue.cpp"]:
        src = os.path.join(CSRC if name in CPP else HERE, name)
        obj = os.path.join(BUILD, name[:-4] + ".o")
        procs.append((subprocess.Popen(flags + ["-c", src, "-o", obj]), name))
        objs.append(obj)
    failed = [n for p, n in procs if p.wait() != 0]
    if failed:
        raise RuntimeError("emulated build failed: " + ", ".join(failed))
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-o", NCCL_OUT, os.path.join(HERE, "nccl_emu.cpp"), "-lpthread"])
    subprocess.check_call(["g++", "-shared", "-o", OUT] + objs + ["-ldl", "-lpthread"])
    return OUT


if __name__ == "__main__":
    print(build(force=True))
