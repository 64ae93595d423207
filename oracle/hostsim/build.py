"""TEST INFRASTRUCTURE ONLY -- builds ``oracle/_build/hostsim/libparcels_b200_hostsim.so``: the product's CUDA sources
(``parcels_b200/csrc``) compiled for the HOST with g++, behind the product's own C-ABI.

How: the sources are copied to ``oracle/_build/hostsim/src`` with two mechanical rewrites --
  * ``kernel<<<grid, block, smem, stream>>>(args);``  ->  ``HS_LAUNCH((kernel), grid, block, smem, stream, args);``
  * the ``extern __shared__ ... pb_smem[];`` declarations are dropped (the shim defines the buffer),
and the three block-cooperative selection kernels of engine.cu (``__syncthreads_count`` / ``__ballot_sync`` scans, which
cannot run one thread at a time) get per-block host equivalents injected next to them -- then compiled against
``oracle/hostsim/include/cuda_runtime.h`` (a stand-in for the CUDA runtime: malloc for device memory, one thread at a time).

The product never builds, loads or links this library; it only answers when ``PB_HOSTSIM_TEST=1`` is set (the test harness
does that) and reports a device named "hostsim".  It exists so that ``pytest -m "not gpu"`` can run the GPU parity tests
against the kernels' SOURCE on machines without a GPU (``tests/test_hostsim_cpu.py``).
"""

from __future__ import annotations

import os
import re
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
CSRC = os.path.join(ROOT, "parcels_b200", "csrc")
OUTDIR = os.path.join(ROOT, "oracle", "_build", "hostsim")
OUT = os.path.join(OUTDIR, "libparcels_b200_hostsim.so")
SOURCES = ["engine.cu", "afast.cu", "agrid.cu", "aslip.cu", "rk45.cu", "advdiff.cu", "hashbuild.cu", "cgrid.cu", "curva.cu"]
HEADERS = ["common.cuh", "agrid.cuh", "rk45.cuh", "cgrid.cuh"]
DEFINES = ["-DPB_SMEM_CACHE", "-DPB_MINBLOCKS=4"]
BLOCK_KERNELS = {"sel_count": "hs_sel_count", "sel_scan": "hs_sel_scan", "sel_scatter": "hs_sel_scatter"}

# per-BLOCK host equivalents of the cooperative selection kernels (engine.cu: sel_count / sel_scan / sel_scatter)
INJECT_AFTER = "// compacted copies of the written columns"
INJECT = r"""
// ---- hostsim: per-block host equivalents of the three cooperative kernels above (called once per block) ----
static void hs_sel_count(ParticlesDev P, SelectRule r, unsigned int* block_counts) {
    unsigned c = 0;
    for (int t = 0; t < SEL_BLOCK; ++t) {
        const long long i = (long long)blockIdx.x * SEL_BLOCK + t;
        c += (i < P.n && sel_flag(P, r, i)) ? 1u : 0u;
    }
    block_counts[blockIdx.x] = c;
}
static void hs_sel_scan(const unsigned int* block_counts, long long* block_offsets, long long nb, long long* total) {
    long long acc = 0;
    for (long long i = 0; i < nb; ++i) { block_offsets[i] = acc; acc += (long long)block_counts[i]; }
    *total = acc;
}
static void hs_sel_scatter(ParticlesDev P, SelectRule r, const long long* block_offsets, long long* idx) {
    long long k = block_offsets[blockIdx.x];
    for (int t = 0; t < SEL_BLOCK; ++t) {
        const long long i = (long long)blockIdx.x * SEL_BLOCK + t;
        if (i < P.n && sel_flag(P, r, i)) idx[k++] = i;
    }
}
"""


def _balanced(text: str, start: int) -> int:
    """index just past the parenthesis that closes the one opened at text[start]"""
    depth = 0
    for i in range(start, len(text)):
        if text[i] == "(":
            depth += 1
        elif text[i] == ")":
            depth -= 1
            if depth == 0:
                return i + 1
    raise ValueError("unbalanced launch arguments")


def rewrite(text: str) -> str:
    text = re.sub(r"^[ \t]*extern __shared__[^\n]*pb_smem\[\];[ \t]*\n", "", text, flags=re.M)
    text = text.replace("__noinline__", "HS_NOINLINE")  # `__noinline__` is a reserved attribute spelling inside libstdc++
    out, pos = [], 0
    for m in re.finditer(r"([A-Za-z_][\w]*(?:<[^;{}]*?>)?)\s*<<<(.*?)>>>\s*\(", text, flags=re.S):
        if m.start() < pos:
            continue
        end = _balanced(text, m.end() - 1)
        kernel, cfg, args = m.group(1), m.group(2), text[m.end() : end - 1]
        name = kernel.split("<")[0]
        macro, target = ("HS_LAUNCH_BLOCKS", BLOCK_KERNELS[name]) if name in BLOCK_KERNELS else ("HS_LAUNCH", kernel)
        out.append(text[pos : m.start()])
        out.append(f"{macro}(({target}), {cfg}, {args})")
        pos = end
    out.append(text[pos:])
    text = "".join(out)
    if INJECT_AFTER in text:
        text = text.replace(INJECT_AFTER, INJECT + INJECT_AFTER, 1)
    return text


def needs_build() -> bool:
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    deps = [os.path.join(CSRC, f) for f in SOURCES + HEADERS] + [__file__, os.path.join(ROOT, "include", "parcels_b200.h")]
    for d, _, fs in os.walk(os.path.join(HERE, "include")):
        deps += [os.path.join(d, f) for f in fs]
    return any(os.path.getmtime(f) > t for f in deps)


def build(force: bool = False) -> str:
    if not force and not needs_build():
        return OUT
    src = os.path.join(OUTDIR, "src")
    shutil.rmtree(src, ignore_errors=True)
    os.makedirs(src)
    n_launch = 0
    for f in SOURCES + HEADERS:
        text = open(os.path.join(CSRC, f)).read()
        new = rewrite(text)
        n_launch += new.count("HS_LAUNCH")
        new = new.replace('#include "../../include/parcels_b200.h"', f'#include "{os.path.join(ROOT, "include", "parcels_b200.h")}"')
        open(os.path.join(src, f.replace(".cu", ".cpp") if f.endswith(".cu") else f), "w").write(new)
    assert n_launch == sum(open(os.path.join(CSRC, f)).read().count("<<<") for f in SOURCES), "a kernel launch was not rewritten"
    cxx = os.environ.get("CXX", "g++")
    flags = ["-O1", "-std=c++17", "-fPIC", "-ffp-contract=off", "-w", "-I", os.path.join(HERE, "include"), *DEFINES]
    procs = []
    for f in SOURCES:
        cpp = os.path.join(src, f.replace(".cu", ".cpp"))
        obj = cpp.replace(".cpp", ".o")
        cmd = [cxx, *flags, "-c", "-o", obj, cpp]
        procs.append((cmd, obj, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)))
    objs = []
    for cmd, obj, p in procs:
        o, e = p.communicate()
        if p.returncode != 0:
            raise RuntimeError(f"hostsim compile failed:\n{' '.join(cmd)}\n{o}\n{e[:6000]}")
        objs.append(obj)
    res = subprocess.run([cxx, "-shared", "-o", OUT, *objs, "-ldl"], capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError(f"hostsim link failed:\n{res.stdout}\n{res.stderr[:4000]}")
    return OUT


if __name__ == "__main__":
    print(build(force=True))
