"""The 64-output-channel instances of the two-limb conv (tc_conv_x3_kernel<64, ...>) compute the transposed tile
D^T[co][pos] = W . X^T: one m64n128k16 per k-step (2 KB of weights + 4 KB of activation rows from shared memory per 131 072
MACs) instead of two m64n64k16 (4 KB + 4 KB), which at tensor peak would need all of the SM's shared-memory bandwidth for
the operand reads alone.  This compiles conv_x3.cu exactly as the library build does and checks, per instance, that the
SASS issues only 64x128x16 HGMMAs and that the transposed epilogue does not spill more than the untransposed one did."""
import os
import re
import shutil
import subprocess

import pytest

from unsuperviseddeephomographyral2018_b200 import build_ext

# tc_conv_x3_kernel<N_OUT, CB, T, FMT_A, FMT_W, FMT_O, ROWS>
INSTANCE = re.compile(r"_ZN3udh2tc17tc_conv_x3_kernelILi(\d+)ELi(\d+)ELi(\d+)ELi-?\d+ELi-?\d+ELi-?\d+ELi(\d+)EEEv\w*")
# spill bytes (stores) of the untransposed kernels, keyed by (CB, T, ROWS)
MAX_SPILL = {(1, 2, 0): 8, (2, 2, 0): 8, (1, 2, 2): 8, (1, 2, 1): 60}


def _tool(name):
    p = os.path.join(os.path.dirname(os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")), name)
    return p if os.path.exists(p) else shutil.which(name)


@pytest.mark.skipif(_tool("nvcc") is None or _tool("cuobjdump") is None, reason="the CUDA toolkit is not installed")
def test_conv_x3_64_out_issues_n128_without_more_spills(tmp_path):
    obj = str(tmp_path / "conv_x3.o")
    cmd = [_tool("nvcc")] + build_ext.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build_ext.CSRC, "conv_x3.cu"), "-o", obj]
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert p.returncode == 0, p.stdout
    spills, current = {}, None
    for line in p.stdout.splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", line)
        if m:
            current = m.group(1)
            continue
        m = re.search(r"(\d+) bytes spill stores", line)
        if m and current:
            spills[current] = int(m.group(1))
            current = None
    sass = subprocess.run([_tool("cuobjdump"), "-sass", obj], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                          timeout=300)
    assert sass.returncode == 0, sass.stdout
    hgmma = {}
    fn = None
    for line in sass.stdout.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            fn = m.group(1)
            hgmma[fn] = set()
            continue
        m = re.search(r"HGMMA\.(\d+x\d+x\d+)", line)
        if m and fn:
            hgmma[fn].add(m.group(1))
    checked = set()
    for name, shapes in hgmma.items():
        m = INSTANCE.fullmatch(name)
        if not m or int(m.group(1)) != 64:
            continue
        key = (int(m.group(2)), int(m.group(3)), int(m.group(4)))
        checked.add(key)
        assert shapes == {"64x128x16"}, (name, sorted(shapes))
        assert name in spills, "ptxas -v printed no report for %s" % name
        assert spills[name] <= MAX_SPILL[key], (name, spills[name], MAX_SPILL[key])
    # the generic instances (conv2_x, conv3_1 dgrad) and both row-tile kernels of conv1_2
    assert checked == set(MAX_SPILL), sorted(checked)
