"""One tuning variant of the library: recompile some translation units with other flags, link with the default objects.
   python scripts/build_variant.py cg3 cgrid.cu:-DPB_MINBLOCKS=3 [afast.cu:"-DPB_BLOCK=384 -DPB_MINBLOCKS=1" ...]
   -> parcels_b200/lib/libparcels_b200_<tag>.so   (use with PB_LIB=...)"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from parcels_b200 import build as b  # noqa: E402

b.build()
tag, specs = sys.argv[1], dict(s.split(":", 1) for s in sys.argv[2:])
objdir = os.path.join(b.HERE, "lib", "obj")
objs = []
for src in b.SOURCES:
    obj = os.path.join(objdir, src.replace(".cu", ".o"))
    if src in specs:
        obj = os.path.join(objdir, src.replace(".cu", f"_{tag}.o"))
        base = [f for f in b.EXTRA_FLAGS.get(src, []) if not any(f.split("=")[0] == g.split("=")[0] for g in specs[src].split())]
        cmd = ["nvcc", *b.NVCC_FLAGS, *base, *specs[src].split(), "-Xptxas", "-v", "-c", "-o", obj, os.path.join(b.CSRC, src)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode:
            sys.exit(r.stderr[-3000:])
        lines = r.stderr.splitlines()
        for i, ln in enumerate(lines):
            if "Function properties for _Z13advect_kernel" in ln and ("AFast" in ln and "Li3ELb1EELb0" in ln or "CurvPolicyIffLi2ELb1ELi0" in ln):
                print(f"[{tag} {src}]", ln.split("for ")[1][:60], lines[i + 1].strip(), "|", lines[i + 2].strip().replace("ptxas info    : ", ""))
    objs.append(obj)
out = os.path.join(b.HERE, "lib", f"libparcels_b200_{tag}.so")
subprocess.run(["nvcc", "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", out, *objs, "-ldl"], check=True)
print(out)
