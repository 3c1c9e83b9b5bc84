"""Host side of the ResNet x-vector's masked batches: the per-stage length rule the handle and its twin use against the
output sizes of torch.nn.Conv2d, and the ctypes mirror of xvb_conv2d_args_t (with its lengths field) against the header
as a C compiler lays it out.  CPU only."""
import ctypes as C
import os
import shutil
import subprocess

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("k", [1, 3])
@pytest.mark.parametrize("stride", [1, 2])
def test_level_rule_matches_conv2d_output_sizes(k, stride):
    """L' = (L + 2 pad - k) / s + 1 with pad = k / 2 (conv2d.cu), and ceil(L / 2) per stride-2 stage
    ((L - 1) // 2 + 1, the handle's table), for the 3x3 convs and the 1x1 downsample alike."""
    conv = torch.nn.Conv2d(1, 1, k, stride=stride, padding=k // 2, bias=False)
    for L in range(1, 301):
        with torch.no_grad():
            out = conv(torch.zeros(1, 1, 4, L)).shape[-1]
        assert out == (L + 2 * (k // 2) - k) // stride + 1 == (L - 1) // stride + 1, (k, stride, L)


def test_conv2d_args_mirror_matches_the_header(tmp_path):
    from asv_subtools_b200 import _lib
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    names = [n for n, _ in _lib.Conv2dArgs._fields_]
    assert names[-1] == "lengths"
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "xvb200.h"\nint main(void) {\n'
                   '  printf("%zu\\n", sizeof(xvb_conv2d_args_t));\n' +
                   "".join('  printf("%zu\\n", offsetof(xvb_conv2d_args_t, {}));\n'.format(n) for n in names) + "  return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.check_call([cc, "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)], text=True).split()]
    want = [C.sizeof(_lib.Conv2dArgs)] + [getattr(_lib.Conv2dArgs, n).offset for n in names]
    assert got == want
