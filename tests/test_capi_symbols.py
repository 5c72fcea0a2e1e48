"""The C-ABI library builds, loads on a CPU-only box and exports every symbol include/monorec_b200.h declares."""
import re
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent


def declared_symbols():
    text = (ROOT / "include" / "monorec_b200.h").read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(mr_[a-z0-9_]+)\s*\(", text)))


def test_header_symbols_are_exported_and_bound():
    from monorec_b200 import _lib
    lib = _lib.load()
    names = declared_symbols()
    assert len(names) >= 6
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/monorec_b200.h but not exported"
        assert n in _lib.SIGNATURES, f"{n} has no ctypes signature in monorec_b200/_lib.py"
    assert set(_lib.SIGNATURES) == set(names)


def test_version_and_error_string_without_gpu():
    from monorec_b200 import _lib
    lib = _lib.load()
    assert lib.mr_version() >= 0x100
    assert isinstance(lib.mr_last_error(), bytes)
    # argument validation happens before any CUDA call, so it can be exercised on a CPU-only box
    rc = lib.mr_cost_volume_fwd(None, None, None, None, None, None, 1, 1, 32, 64, 64, 10.0, None, None)
    assert rc == -1 and b"null pointer" in lib.mr_last_error()
    assert lib.mr_cost_volume_host_workspace(8, 4, 32, 256, 512) > 8 * 5 * 32 * 256 * 512 * 4
    assert lib.mr_cost_volume_host_workspace(0, 4, 32, 256, 512) == 0


def test_product_never_imports_oracle():
    """The oracle is test infrastructure: nothing under monorec_b200/ may import it (tier rule 3)."""
    pat = re.compile(r"^\s*(from|import)\s+oracle\b", re.M)
    for p in (ROOT / "monorec_b200").rglob("*.py"):
        assert not pat.search(p.read_text()), f"{p} imports the oracle"


def test_header_is_plain_c_and_a_c_consumer_links(tmp_path):
    """include/monorec_b200.h compiles as C99 (-pedantic) and a C program links against the library and reaches the
    argument checks without a GPU (no compute call)."""
    import shutil
    import subprocess
    from pathlib import Path
    import pytest
    from monorec_b200 import _lib
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    _lib.load()
    root = Path(__file__).resolve().parent.parent
    src = tmp_path / "consumer.c"
    src.write_text('#include "monorec_b200.h"\n#include <stdio.h>\n#include <string.h>\n'
                   'int main(void) {\n'
                   '    mr_conv_desc d; memset(&d, 0, sizeof d);\n'
                   '    if (mr_sizeof_conv_desc() != (int)sizeof d) return 2;\n'
                   '    if (mr_conv2d_nhwc_tc(0, 16, 32, 0, 0) == MR_OK) return 3;\n'
                   '    if (strstr(mr_last_error(), "null descriptor") == 0) return 4;\n'
                   '    if (mr_cost_volume_host_workspace(8, 4, 32, 256, 512) <= 0) return 5;\n'
                   '    {   /* pack a 3x3 layer with two concatenated sources for the half tensor-core path, on the host */\n'
                   '        static float w[24 * 96 * 9]; static unsigned short packed[9 * 32 * 128];\n'
                   '        int src_c[2] = {32, 64}, n_pad = 0, k_pad = 0, i;\n'
                   '        for (i = 0; i < 24 * 96 * 9; ++i) w[i] = (float)(i % 7) - 3.0f;\n'
                   '        if (mr_pack_conv_weights_bytes(24, 2, src_c, 3, 3, MR_DT_F16, &n_pad, &k_pad) != (long long)sizeof packed) return 6;\n'
                   '        if (n_pad != 32 || k_pad != 128) return 7;\n'
                   '        if (mr_pack_conv_weights(w, 24, 2, src_c, 3, 3, MR_DT_F16, packed) != MR_OK) return 8;\n'
                   '        /* tap (1,1), output channel 5, input channel 40 (second source) lives at [4][5][64 + 8]; w = -3 .. 3 */\n'
                   '        if (packed[(4 * 32 + 5) * 128 + 72] != 0xC000 /* half -2.0 = w[(5*96+40)*9+4] = (4684 % 7) - 3 */) return 9;\n'
                   '        if (packed[(4 * 32 + 5) * 128 + 40] != 0) return 10;   /* padding of the first source */\n'
                   '        if (mr_conv_workspace_bytes(&d) != 0) return 11;\n'
                   '    }\n'
                   '    printf("%d\\n", mr_version());\n    return 0;\n}\n')
    exe = tmp_path / "consumer"
    libdir = _lib.LIB_PATH.parent
    subprocess.run(["gcc", "-std=c99", "-pedantic", "-Wall", "-Werror", f"-I{root / 'include'}", str(src), "-o", str(exe),
                    f"-L{libdir}", f"-l:{_lib.LIB_PATH.name}", f"-Wl,-rpath,{libdir}"], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    assert out.returncode == 0, (out.returncode, out.stdout, out.stderr)
    assert int(out.stdout.strip()) == _lib.load().mr_version()


def _header_struct_fields(name):
    text = re.sub(r"/\*.*?\*/", "", (ROOT / "include" / "monorec_b200.h").read_text(), flags=re.S)
    body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (name, name), text, flags=re.S).group(1)
    fields = []
    for decl in body.split(";"):
        decl = re.sub(r"\[.*?\]", "", decl).strip()
        if decl:
            fields += [re.search(r"(\w+)\s*$", part).group(1) for part in decl.split(",")]
    return fields


def test_ctypes_structs_mirror_the_header():
    """ConvDesc / TcPlan list the fields of mr_conv_desc / mr_tc_plan in the header's order (and ConvDesc has its size)."""
    import ctypes
    from monorec_b200 import _lib
    from monorec_b200.conv import ConvDesc, TcPlan
    for cname, cls in (("mr_conv_desc", ConvDesc), ("mr_tc_plan", TcPlan)):
        assert [f for f, _ in cls._fields_] == _header_struct_fields(cname), cname
    assert all(t is ctypes.c_int for _, t in TcPlan._fields_)
    assert ctypes.sizeof(ConvDesc) == _lib.load().mr_sizeof_conv_desc()


# ---- descriptor validation of the convolution entry points, on fake (never dereferenced) 16-byte-aligned pointers -------
def _tc_descs(n=1):
    """n phase descriptors of a valid 3x3 fp32 layer (32 -> 24 channels, 8 x 16, n_pad 32, k_pad 32): never launched."""
    from monorec_b200.conv import ConvDesc
    descs = (ConvDesc * n)()
    for i, d in enumerate(descs):
        d.n_src, d.src[0], d.src_c[0] = 1, 0x7F0000100000, 32
        d.B, d.Hs, d.Ws, d.upsample2 = 1, 8, 16, 0
        d.kh, d.kw, d.sy, d.sx, d.pad_t, d.pad_l = 3, 3, 1, 1, 1, 1
        d.Ho, d.Wo, d.Cout = 8, 16, 24
        d.weight, d.bias, d.dst = 0x7F0000200000 + 0x10000 * i, None, 0x7F0000300000
        d.dst_H, d.dst_W, d.dst_c, d.dst_coff = 8 * n, 16, 24, 0
        d.oy_step, d.ox_step, d.oy_off, d.ox_off = n, 1, i, 0
        d.act, d.act_a, d.act_b, d.src_dtype, d.dst_dtype = 1, 0.1, 1.0, 0, 0
    return descs


def _set(descs, **kw):
    for k, v in kw.items():
        phase = 0
        if k.endswith("_p1"):
            k, phase = k[:-3], 1
        if k in ("src", "src_c"):
            getattr(descs[phase], k)[0] = v
        else:
            setattr(descs[phase], k, v)
    return descs


# (descriptor changes, n_pad, k_pad, n_phases, text the error message must contain)
BAD_TC = [
    (dict(oy_off=-1), 32, 32, 1, "oy_off"),
    (dict(ox_off=-3), 32, 32, 1, "ox_off"),
    (dict(oy_off_p1=-1), 32, 32, 2, "oy_off"),
    (dict(act=4), 32, 32, 1, "act"),
    (dict(act=-1), 32, 32, 1, "act"),
    (dict(oy_step=0), 32, 32, 1, "oy_step"),
    (dict(ox_step=-1), 32, 32, 1, "ox_step"),
    (dict(src_dtype=2), 32, 32, 1, "src_dtype"),
    (dict(dst_dtype=5), 32, 32, 1, "dst_dtype"),
    (dict(src_c=30), 32, 32, 1, "src_c"),
    (dict(src_dtype=1, src_c=36), 32, 64, 1, "src_c"),
    (dict(src=0x7F0000100004), 32, 32, 1, "aligned"),
    (dict(src=None), 32, 32, 1, "source 0"),
    (dict(weight=0x7F0000200008), 32, 32, 1, "weight"),
    (dict(weight_p1=None), 32, 32, 2, "weight"),
    (dict(), 32, 64, 1, "k_pad"),
    (dict(src_dtype=1), 32, 64 + 32, 1, "k_pad"),
    (dict(), 24, 32, 1, "n_pad"),
    (dict(Cout=300, dst_c=300), 32, 32, 1, "Cout"),
    (dict(dst_coff=-1), 32, 32, 1, "dst_coff"),
    (dict(dst_coff=1), 32, 32, 1, "dst_coff"),
    (dict(upsample2=1), 32, 32, 1, "upsample2"),
    (dict(n_src=0), 32, 32, 1, "n_src"),
    (dict(n_src=4), 32, 32, 1, "n_src"),
    (dict(sy=5), 32, 32, 1, "sy"),
    (dict(kw_p1=0), 32, 32, 2, "kw"),
    (dict(Ho=9), 32, 32, 1, "placement"),
    (dict(ox_off_p1=1), 32, 32, 2, "placement"),
    (dict(dst=None), 32, 32, 1, "dst"),
    (dict(dst_c_p1=32), 32, 32, 2, "differs"),
]


def test_tc_descriptor_validation_without_gpu():
    """Every bad field of a tensor-core descriptor is rejected with MR_EINVAL and a message naming it, before any CUDA call
    (also in the plan query); negative output offsets in the CUDA-core entry point too.  A valid descriptor gets past
    validation: the plan query then reports a plan (GPU) or a CUDA error (no GPU), never MR_EINVAL."""
    import ctypes
    from monorec_b200 import _lib
    from monorec_b200.conv import TcPlan
    lib = _lib.load()
    plan = TcPlan()
    rc = lib.mr_conv2d_nhwc_tc_plan(_tc_descs(2), 2, 32, 32, ctypes.byref(plan))
    assert rc != -1, lib.mr_last_error()
    if rc == 0:
        assert plan.kernel == 0 and plan.n_pad == 32 and plan.total_tiles == 2
    for changes, n_pad, k_pad, n_phases, text in BAD_TC:
        descs = _set(_tc_descs(n_phases), **changes)
        if n_phases == 1:
            rc = lib.mr_conv2d_nhwc_tc(descs, n_pad, k_pad, 1, None)
        else:
            rc = lib.mr_conv2d_nhwc_tc_phases(descs, n_phases, n_pad, k_pad, 1, None)
        msg = lib.mr_last_error().decode()
        assert rc == -1 and text in msg, (changes, rc, msg)
        rc = lib.mr_conv2d_nhwc_tc_plan(_set(_tc_descs(n_phases), **changes), n_phases, n_pad, k_pad, ctypes.byref(plan))
        assert rc == -1 and text in lib.mr_last_error().decode(), (changes, rc)
    assert lib.mr_conv2d_nhwc_tc_plan(_tc_descs(1), 1, 32, 32, None) == -1
    for changes in (dict(oy_off=-1), dict(ox_off=-1)):
        d = _set(_tc_descs(1), **changes)
        d[0].weight = 0x7F0000200000                       # [kh][kw][Cin][Cout] fp32 on this path (never read)
        assert lib.mr_conv2d_nhwc(d, None) == -1 and next(iter(changes)) in lib.mr_last_error().decode()
