"""Half-precision cost volumes (volume_dtype=torch.float16): the parts that need no GPU.

The C ABI's argument checks of the half entries (fake, never dereferenced pointers), the workspace sizes of the half host
entry, the Python keyword and its validation, and a C consumer of the new declarations.  The GPU side is
tests/test_cv_half_gpu.py.
"""
import ctypes
import inspect

import pytest
import torch

FRAMES = (ctypes.c_void_p * 8)(*[0x7F0000400000 + 0x100000 * i for i in range(8)])
KEY, PROJ, Z, PZ, CV, SF, NHWC = (0x7F0000100000, 0x7F0000200000, 0x7F0000300000, 0x7F0000380000, 0x7F0001000000,
                                  0x7F0002000000, 0x7F0003000000)


def _lib():
    from monorec_b200 import _lib
    return _lib.load()


def test_typed_entry_validation_without_gpu():
    """Bad arguments of mr_cost_volume_fwd_typed give MR_EINVAL (MR_ENOSUPPORT for the plain L1 difference) and a message
    naming the field, before any CUDA call."""
    lib = _lib()

    def call(depths=Z, pixel=None, cv=CV, sf=SF, nhwc=None, nhwc_dtype=0, F=2, D=32, matching=1, centered=1, out_dtype=1):
        rc = lib.mr_cost_volume_fwd_typed(KEY, FRAMES, PROJ, depths, pixel, cv, sf, nhwc, nhwc_dtype, 1, F, D, 64, 64, 10.0,
                                          None, matching, centered, out_dtype, None)
        return rc, lib.mr_last_error().decode()

    rc, msg = call(matching=0)
    assert rc == -2 and "matching" in msg, (rc, msg)
    cases = [(dict(out_dtype=2), "out_dtype"), (dict(out_dtype=-1), "out_dtype"), (dict(matching=4), "matching"),
             (dict(centered=2), "centered"), (dict(pixel=PZ), "pixel_depths"), (dict(depths=None), "pixel_depths"),
             (dict(depths=None, pixel=PZ + 2), "pixel_depths"), (dict(D=1), "D="), (dict(D=129), "D="), (dict(F=0), "F="),
             (dict(F=9), "F="), (dict(nhwc=NHWC, nhwc_dtype=2), "nhwc_dtype"), (dict(cv=None), "out_cv"),
             (dict(sf=None), "out_sfcv"), (dict(cv=CV + 2), "out_cv"), (dict(sf=SF + 2), "out_sfcv"),
             (dict(cv=CV + 4, out_dtype=0), "out_cv"), (dict(sf=SF + 4, out_dtype=0), "out_sfcv")]
    for kw, text in cases:
        rc, msg = call(**kw)
        assert rc == -1 and text in msg and "mr_cost_volume_fwd_typed" in msg, (kw, rc, msg)


def test_half_host_entry_sizes_and_validation_without_gpu():
    lib = _lib()
    B, F, D, H, W = 8, 4, 32, 256, 512
    ws32, ws16 = lib.mr_cost_volume_host_workspace(B, F, D, H, W), lib.mr_cost_volume_host_f16_workspace(B, F, D, H, W)
    vol = (F + 1) * B * D * H * W
    # the images stay fp32; the two volumes take half the bytes
    assert ws16 >= vol * 2 and ws32 - ws16 >= vol * 2
    assert lib.mr_cost_volume_host_f16_sfcv_offset(B, F, D, H, W) >= B * D * H * W * 2
    assert lib.mr_cost_volume_host_f16_sfcv_offset(B, F, D, H, W) < lib.mr_cost_volume_host_sfcv_offset(B, F, D, H, W)
    assert lib.mr_cost_volume_host_f16_workspace(0, F, D, H, W) == 0
    assert lib.mr_cost_volume_host_f16_sfcv_offset(B, F, 1, H, W) == -1
    h = 0x7F0005000000
    args = [h] * 8 + [B, F, D, H, W, 0.0025, 0.33, 10.0]
    assert lib.mr_cost_volume_host_f16(*([h] * 6 + [None, h]), B, F, D, H, W, 0.0025, 0.33, 10.0, h, ws16) == -1
    assert b"mr_cost_volume_host_f16: null pointer" in lib.mr_last_error()
    assert lib.mr_cost_volume_host_f16(*([h] * 8), B, 9, D, H, W, 0.0025, 0.33, 10.0, h, ws16) == -1
    assert b"bad shape" in lib.mr_last_error()
    assert lib.mr_cost_volume_host_f16(*args, h, ws16 - 1) == -3
    assert b"workspace too small" in lib.mr_last_error()


def test_typed_layout_pool_mask_validation_without_gpu():
    """The layout, pooling and masking entries with half tensors (MR_DT_F16 = 1), a dtype argument other than MR_DT_F32 /
    MR_DT_F16, and the channel-vector width that follows the dtype: MR_EINVAL and a message naming the argument, before any
    CUDA call (fake, never dereferenced pointers)."""
    lib = _lib()
    src, dst, m = 0x7F0006000000, 0x7F0007000000, 0x7F0008000000
    assert lib.mr_nchw_to_nhwc(src, 1, dst, 2, 1, 32, 8, 8, 32, 0, None, None) == -1
    assert b"dst_dtype" in lib.mr_last_error()
    assert lib.mr_nchw_to_nhwc(src, 1, dst, 1, 1, 32, 8, 8, 32, 4, None, None) == -1
    assert b"channel slice" in lib.mr_last_error()
    assert lib.mr_nchw_to_nhwc(None, 1, dst, 0, 1, 32, 8, 8, 32, 0, None, None) == -1
    assert lib.mr_mask_volume(src, None, dst, 1, 1, 32, 64, None) == -1
    assert b"mr_mask_volume" in lib.mr_last_error()
    bad_dtype = [(lambda d: lib.mr_nchw_to_nhwc(src, d, dst, 1, 1, 32, 8, 8, 32, 0, None, None), b"mr_nchw_to_nhwc: src_dtype"),
                 (lambda d: lib.mr_nchw_to_nhwc(src, 1, dst, d, 1, 32, 8, 8, 32, 0, None, None), b"mr_nchw_to_nhwc: dst_dtype"),
                 (lambda d: lib.mr_maxpool2_nhwc(src, dst, d, 1, 8, 8, 32, None), b"mr_maxpool2_nhwc: dtype"),
                 (lambda d: lib.mr_max_over_frames(src, dst, d, 2, 64, None), b"mr_max_over_frames: dtype"),
                 (lambda d: lib.mr_mask_volume(src, m, dst, d, 1, 32, 64, None), b"mr_mask_volume: dtype")]
    for call, text in bad_dtype:
        for d in (2, -1):
            assert call(d) == -1 and text in lib.mr_last_error(), (text, d, lib.mr_last_error())
    # 4 channels (values per frame) are one fp32 vector but half a half vector: the fp32 call gets past the width check to
    # the null destination, the half call stops at the width
    for dtype, text in ((0, b"null pointer"), (1, b"C % 8")):
        assert lib.mr_maxpool2_nhwc(src, None, dtype, 1, 8, 8, 4, None) == -1
        assert text in lib.mr_last_error(), (dtype, lib.mr_last_error())
    for dtype, text in ((0, b"null pointer"), (1, b"multiple of 8")):
        assert lib.mr_max_over_frames(src, None, dtype, 2, 4, None) == -1
        assert text in lib.mr_last_error(), (dtype, lib.mr_last_error())


def test_volume_dtype_keyword():
    from monorec_b200.cost_volume import CostVolumeModule
    from monorec_b200.model import MonoRecModel
    for cls in (CostVolumeModule, MonoRecModel):
        params = list(inspect.signature(cls.__init__).parameters.values())
        assert params[-1].name == "volume_dtype" and params[-1].default is torch.float32, cls
    assert CostVolumeModule().volume_dtype is torch.float32
    assert CostVolumeModule(volume_dtype=torch.float16).volume_dtype is torch.float16
    assert CostVolumeModule(use_ssim=2, not_center_cv=True, volume_dtype=torch.float16).volume_dtype is torch.float16
    for bad in (torch.bfloat16, torch.float64, torch.int16, "float16", None, 16):
        with pytest.raises(ValueError, match="volume_dtype"):
            CostVolumeModule(volume_dtype=bad)
    m = MonoRecModel()
    assert m.volume_dtype is torch.float32 and m.cv_module.volume_dtype is torch.float32
    m = MonoRecModel(volume_dtype=torch.float16)
    assert m.volume_dtype is torch.float16 and m.cv_module.volume_dtype is torch.float16
    with pytest.raises(ValueError, match="volume_dtype"):
        MonoRecModel(volume_dtype=torch.bfloat16)


def test_c_consumer_of_the_typed_entries(tmp_path):
    """The half-volume declarations and the typed layout / masking entries compile as C99 (-pedantic) and link; their
    argument checks answer without a GPU."""
    import shutil
    import subprocess
    from pathlib import Path
    from monorec_b200 import _lib
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    _lib.load()
    root = Path(__file__).resolve().parent.parent
    src = tmp_path / "consumer_f16.c"
    src.write_text('#include "monorec_b200.h"\n#include <string.h>\n'
                   'int main(void) {\n'
                   '    long long w32 = mr_cost_volume_host_workspace(2, 2, 32, 64, 128);\n'
                   '    long long w16 = mr_cost_volume_host_f16_workspace(2, 2, 32, 64, 128);\n'
                   '    if (w16 <= 0 || w16 >= w32) return 2;\n'
                   '    if (mr_cost_volume_host_f16_sfcv_offset(2, 2, 32, 64, 128) <= 0) return 3;\n'
                   '    if (mr_cost_volume_fwd_typed(0, 0, 0, 0, 0, 0, 0, 0, MR_DT_F32, 1, 2, 32, 64, 64, 10.0f, 0, MR_CV_SSIM, 1,\n'
                   '                                 7, 0) != MR_EINVAL) return 4;\n'
                   '    if (strstr(mr_last_error(), "out_dtype") == 0) return 5;\n'
                   '    if (mr_cost_volume_host_f16(0, 0, 0, 0, 0, 0, 0, 0, 2, 2, 32, 64, 128, 0.0025f, 0.33f, 10.0f, 0, w16)\n'
                   '        != MR_EINVAL) return 6;\n'
                   '    if (mr_mask_volume(0, 0, 0, MR_DT_F16, 1, 1, 1, 0) != MR_EINVAL) return 7;\n'
                   '    if (mr_nchw_to_nhwc(0, MR_DT_F16, 0, MR_DT_F16, 1, 1, 1, 1, 1, 0, 0, 0) != MR_EINVAL) return 8;\n'
                   '    return 0;\n}\n')
    exe = tmp_path / "consumer_f16"
    libdir = _lib.LIB_PATH.parent
    subprocess.run(["gcc", "-std=c99", "-pedantic", "-Wall", "-Werror", f"-I{root / 'include'}", str(src), "-o", str(exe),
                    f"-L{libdir}", f"-l:{_lib.LIB_PATH.name}", f"-Wl,-rpath,{libdir}"], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    assert out.returncode == 0, (out.returncode, out.stdout, out.stderr)
