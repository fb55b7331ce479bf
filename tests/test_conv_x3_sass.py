"""The two-limb conv kernel, tc_conv_x3_kernel, runs four warpgroups: producers, two MMA warpgroups and an epilogue
warpgroup that drains each item's accumulators from shared memory while the MMA warpgroups start the next item.  Its 512
threads share the register file through setmaxnreg: 40 (producers) + 112 (epilogue) + 2 x 176 (MMA) <= 512 registers per
thread-quad.  The 64-output-channel instances compute the transposed tile D^T[co][pos] = W . X^T: one m64n128k16 per k-step
(2 KB of weights + 4 KB of activation rows from shared memory per 131 072 MACs) instead of two m64n64k16 (4 KB + 4 KB), which
at tensor peak would need all of the SM's shared-memory bandwidth for the operand reads alone.  This compiles conv_x3.cu
exactly as the library build does and checks, per instance, that the SASS applies that register split, issues only
64x128x16 HGMMAs with one wgmma group left in flight (WARPGROUP.DEPBAR.LE gsb0, 0x1), that ptxas reports no serialised
wgmma (C7510 / C7519) and that the spills stay where they are."""
import os
import re
import shutil
import subprocess

import pytest

from unsuperviseddeephomographyral2018_b200 import build_ext

# tc_conv_x3_kernel<N_OUT, CB, T, FMT_A, FMT_W, FMT_O, ROWS>
INSTANCE = re.compile(r"_ZN3udh2tc17tc_conv_x3_kernelILi(\d+)ELi(\d+)ELi(\d+)ELi-?\d+ELi-?\d+ELi-?\d+ELi(\d+)EEEv\w*")
# spill bytes (stores) keyed by (N_OUT, CB, T, ROWS): the pooled conv1_2 forward keeps its 32 maxima and routing bits live
# across the lane exchange in the 112-register epilogue warpgroup
MAX_SPILL = {(64, 1, 2, 0): 0, (64, 2, 2, 0): 0, (128, 1, 1, 0): 0, (128, 2, 1, 0): 0, (64, 1, 2, 2): 0, (64, 1, 2, 1): 24}
REGS = {"DEALLOC": {0x28, 0x70}, "TRY_ALLOC": {0xB0}}   # producers 40, epilogue 112 | MMA 176


def _tool(name):
    p = os.path.join(os.path.dirname(os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")), name)
    return p if os.path.exists(p) else shutil.which(name)


@pytest.mark.skipif(_tool("nvcc") is None or _tool("cuobjdump") is None, reason="the CUDA toolkit is not installed")
def test_conv_x3_register_split_spills_and_pipelined_hgmma(tmp_path):
    obj = str(tmp_path / "conv_x3.o")
    cmd = [_tool("nvcc")] + build_ext.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build_ext.CSRC, "conv_x3.cu"), "-o", obj]
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert p.returncode == 0, p.stdout
    spills, current = {}, None
    for line in p.stdout.splitlines():
        assert not ("tc_conv_x3_kernel" in line and ("(C7510)" in line or "(C7519)" in line)), line
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
    info, fn = {}, None
    for line in sass.stdout.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            fn = m.group(1)
            info[fn] = {"hgmma": set(), "depbar": set(), "DEALLOC": set(), "TRY_ALLOC": set()}
            continue
        if fn is None:
            continue
        m = re.search(r"HGMMA\.(\d+x\d+x\d+)", line)
        if m:
            info[fn]["hgmma"].add(m.group(1))
        m = re.search(r"WARPGROUP\.DEPBAR\.LE gsb0, (0x[0-9a-f]+)", line)
        if m:
            info[fn]["depbar"].add(int(m.group(1), 16))
        m = re.search(r"USETMAXREG\.(DEALLOC|TRY_ALLOC)\.CTAPOOL (?:UP\d+, )?(0x[0-9a-f]+)", line)
        if m:
            info[fn][m.group(1)].add(int(m.group(2), 16))
    checked = set()
    for name, d in info.items():
        m = INSTANCE.fullmatch(name)
        if not m:
            continue
        key = tuple(int(m.group(i)) for i in range(1, 5))
        checked.add(key)
        assert d["hgmma"] == {"64x128x16"}, (name, sorted(d["hgmma"]))
        assert 1 in d["depbar"], (name, "no wgmma group left in flight", sorted(d["depbar"]))
        assert d["DEALLOC"] == REGS["DEALLOC"] and d["TRY_ALLOC"] == REGS["TRY_ALLOC"], (name, d["DEALLOC"], d["TRY_ALLOC"])
        assert name in spills, "ptxas -v printed no report for %s" % name
        assert spills[name] <= MAX_SPILL[key], (name, spills[name], MAX_SPILL[key])
    # every instance the train step launches: conv2_x, conv3_1 (fwd and dgrad), the 128 -> 128 layers, conv1_2's row tiles
    assert checked == set(MAX_SPILL), sorted(checked)
