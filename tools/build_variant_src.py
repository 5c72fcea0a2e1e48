"""Variant library with another cost_volume.cu: python tools/build_variant_src.py TAG /path/to/cost_volume.cu
-> monorec_b200/variants/libmonorec_b200_TAG.so (load it with MONOREC_B200_LIB=<path>).  The variant is an edited copy of the
source; the package's flags are used unchanged."""
import shutil
import subprocess
import sys
import tempfile
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from monorec_b200 import build as B  # noqa: E402

tag, src = sys.argv[1], Path(sys.argv[2])
out = ROOT / "monorec_b200" / "variants"
out.mkdir(exist_ok=True)
lib = out / f"libmonorec_b200_{tag}.so"
with tempfile.TemporaryDirectory() as td:
    td = Path(td) / "monorec_b200" / "csrc"
    td.mkdir(parents=True)
    (td.parent.parent / "include").mkdir()
    shutil.copy(ROOT / "include" / "monorec_b200.h", td.parent.parent / "include")
    for f in B.CSRC.iterdir():
        shutil.copy(f, td / f.name)
    shutil.copy(src, td / "cost_volume.cu")
    cmd = [B.NVCC, *B.FLAGS, "-shared", "-Xcompiler", "-fPIC", "-Xcompiler", "-O2", "-o", str(lib)] + [str(s) for s in sorted(td.glob("*.cu"))]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        sys.exit(1)
print(lib)
