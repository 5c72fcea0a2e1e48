"""Per-row-step SASS opcode mix of the cost-volume kernel's hot loops, from the compiled code alone (no GPU needed).

    python tools/sass_loop_mix.py [--build] [path/to/cost_volume.cu]

Compiles cost_volume.cu (default: the package's) for sm_90a with the library's flags into a temporary cubin, disassembles
it with line information and finds the loops of cost_volume_kernel (backward branches).  A loop is attributed to a
call site of march_unit<MODE> or pixel_phase<T> when the inlining chains of its instructions reach that call's source
line.  For each march mode it prints the largest such loop, the row loop (three row steps per body), and for the
per-pixel phase its loops; counts are per row step for the march and per loop iteration otherwise.

The kernel is instantiated as cost_volume_kernel<PIX, ERR, CENTER, OUT, NC>: depth source (plane table / per-pixel
cv_depths), error mode (1 SSIM, 2 SSIM + L1, 3 box L1: MR_CV_*), centred or uncentred fused volume, the volumes' storage
type (float or __half) and the frames' channel count (3, or 1 for grayscale frames).  The twelve fp32 three-channel
instantiations come first (the two default ones, SSIM centred, plane depths then per-pixel depths, lead), the twelve half
ones after them in the same order, then the same twenty-four with one channel.  A source from before the volume type was a template
parameter is reported under the fp32 titles; one from before the error mode was has only cost_volume_kernel<PIX>, reported
under the first two titles.
"""
import collections
import re
import subprocess
import sys
import tempfile
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from monorec_b200 import build as B  # noqa: E402

GROUPS = [  # (name, opcode prefixes); the first match wins
    ("FFMA", ("FFMA",)), ("FADD", ("FADD",)), ("FMUL", ("FMUL",)), ("FMNMX/FSET", ("FMNMX", "FSET", "FSEL", "FCHK")),
    ("MUFU", ("MUFU",)), ("LDS", ("LDS",)), ("STS", ("STS",)), ("LDG", ("LDG",)), ("STG", ("STG",)),
    ("LDL/STL", ("LDL", "STL")), ("SHFL", ("SHFL",)), ("VOTE", ("VOTE",)),
    ("branch", ("BRA", "BSSY", "BSYNC", "WARPSYNC", "EXIT", "BAR", "NOP")),
    ("int/move", ("IMAD", "IADD", "VIADD", "LEA", "LOP", "SHF", "SEL", "MOV", "ISETP", "IMNMX", "VIMNMX", "PRMT", "P2R", "R2P",
                  "PLOP", "I2F", "F2I", "UMOV", "ULDC", "S2R", "CS2R", "LDC", "UIADD", "ULEA", "USHF", "ULOP", "UISETP", "R2UR")),
]


def group(op):
    for name, prefixes in GROUPS:
        if op.startswith(prefixes):
            return name
    return "other"


def disassemble(src):
    with tempfile.TemporaryDirectory() as td:
        cubin = Path(td) / "cv.cubin"
        flags = [f for f in B.FLAGS if f != "-lineinfo"]
        # (a copy kept elsewhere, e.g. a parent version for comparison, still finds the package's headers)
        inc = ["-I", str(ROOT / "include"), "-I", str(Path(src).resolve().parent), "-I", str(B.CSRC)]
        subprocess.run([B.NVCC, *flags, "-lineinfo", "-cubin", *inc, "-o", str(cubin), str(src)], check=True)
        return subprocess.run([B.NVCC.replace("nvcc", "nvdisasm"), "-c", "-gi", str(cubin)], check=True,
                              capture_output=True, text=True).stdout


ERR_NAMES = {1: "SSIM", 2: "SSIM + L1", 3: "box L1"}
OUT_TYPES = (("f", "float", "fp32"), ("6__half", "__half", "half"))
# (label, mangled template arguments of cost_volume_kernel<PIX, ERR, CENTER, OUT, NC>, then those of older sources: without
# the channel count (three channels), without the volume type (fp32 only), with only <PIX>)
INSTANTIATIONS = [
    (f"{'per-pixel' if pix else 'plane'} depths, {ERR_NAMES[err]}, {'centred' if ctr else 'uncentred'}, {oname} volumes, "
     f"{nc} channel{'s' if nc > 1 else ''} "
     f"(cost_volume_kernel<{'true' if pix else 'false'}, {err}, {'true' if ctr else 'false'}, {otype}, {nc}>)",
     f"cost_volume_kernelILb{pix}ELi{err}ELb{ctr}E{omangled}Li{nc}EEE",
     [f for f in (f"cost_volume_kernelILb{pix}ELi{err}ELb{ctr}E{omangled}EE" if nc == 3 else None,
                  f"cost_volume_kernelILb{pix}ELi{err}ELb{ctr}EE" if nc == 3 and omangled == "f" else None,
                  f"cost_volume_kernelILb{pix}EE" if nc == 3 and err == 1 and ctr and omangled == "f" else None) if f])
    for nc in (3, 1)
    for omangled, otype, oname in OUT_TYPES
    for err, ctr, pix in [(1, 1, 0), (1, 1, 1)] + [(e, c, p) for e in (1, 2, 3) for c in (1, 0) for p in (0, 1)
                                                    if (e, c) != (1, 1)]
]


def kernel_instructions(dis, name="cost_volume_kernelILb0ELi1ELb1EfLi3EEE"):
    """[(addr, opcode, text, source lines of the inlining chain)] and {label: addr} of the kernel whose .text section
    name contains `name` (default: the plane instantiation)."""
    ins, labels, cur, inside, pending = [], {}, [], False, []
    for line in dis.splitlines():
        if line.startswith(".text."):
            inside = name in line
            continue
        if not inside:
            continue
        if line.lstrip().startswith("//##"):
            cur = [int(x) for x in re.findall(r"line (\d+)", line)]
            continue
        m = re.match(r"(\.L_x_\d+):", line.strip())
        if m:
            pending.append(m.group(1))
            continue
        m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;", line)
        if m:
            addr = int(m.group(1), 16)
            for lab in pending:
                labels[lab] = addr
            pending = []
            body = re.sub(r"^@!?U?P\w+\s+", "", m.group(2).strip())
            ins.append((addr, body.split()[0], body, tuple(cur)))
    return ins, labels


def main():
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    src = Path(args[0]) if args else B.CSRC / "cost_volume.cu"
    text = src.read_text().splitlines()
    sites = {}
    for i, l in enumerate(text, 1):
        m = re.search(r"\b(march_unit|pixel_phase)<(\d)(?:, \w+)*>\(", l)
        if m and "__device__" not in l and "void" not in l:
            sites[f"{m.group(1)}<{m.group(2)}>"] = i
    dis = disassemble(src)
    for k, (title, name, older) in enumerate(INSTANTIATIONS):
        if name not in dis:
            found = [o for o in older if o in dis]   # (a source from before a template parameter was added)
            if found:
                name = found[0]
            elif k == 0 and "cost_volume_kernelILb" not in dis:   # (from before the depth source became one)
                report(src, "cost_volume_kernel", *kernel_instructions(dis, "cost_volume_kernel"), sites)
                continue
            else:
                continue
        if k:
            print("\n" + "=" * 100)
        report(src, title, *kernel_instructions(dis, name), sites)


def report(src, title, ins, labels, sites):
    index = {a: k for k, (a, *_r) in enumerate(ins)}
    loops = []
    for k, (addr, op, body, _l) in enumerate(ins):
        if op == "BRA":
            tgt = re.search(r"(\.L_x_\d+)", body)
            if tgt and labels.get(tgt.group(1), addr + 1) <= addr:
                loops.append((index[labels[tgt.group(1)]], k))
    print(f"{src.name}: {title}, {len(ins)} instructions, {len(loops)} loops")
    for name, site in sorted(sites.items(), key=lambda kv: kv[1]):
        mine = []
        for lo, hi in loops:
            # most of the loop's instructions come from this call (ptxas merges a few common tails across call sites)
            if 2 * sum(site in ch for _a, _o, _b, ch in ins[lo:hi + 1]) > hi - lo + 1:
                mine.append((lo, hi))
        if not mine:
            print(f"\n{name} (line {site}): no loop found")
            continue
        picks = [max(mine, key=lambda r: r[1] - r[0])] if name.startswith("march") else sorted(set(mine))
        for lo, hi in picks:
            n = hi - lo + 1
            per = 3 if name.startswith("march") else 1
            mix = collections.Counter(group(o) for _a, o, _b, _c in ins[lo:hi + 1])
            unit = "per row step" if per == 3 else "per iteration"
            print(f"\n{name} (line {site}): loop {ins[lo][0]:#06x}-{ins[hi][0]:#06x}, {n} instructions, "
                  f"{n / per:.1f} {unit}")
            print("  " + ", ".join(f"{g} {c / per:.1f}" for g, c in sorted(mix.items(), key=lambda kv: -kv[1])))


if __name__ == "__main__":
    main()
