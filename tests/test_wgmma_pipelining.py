"""The wgmma kernels only reach tensor-core throughput when each warpgroup keeps several MMAs in flight.  ptxas silently
drops that to one MMA at a time in two situations, and says so only with -Xptxas -v:
  C7510  any function call in the kernel (a device printf is enough) serialises every wgmma of the kernel;
  C7519  a warpgroup.arrive is injected because accumulator registers are used across in-flight MMAs (e.g. a loop
         back-edge between them).
This compiles the two translation units that hold the wgmma kernels exactly as the library build does and fails on either
diagnostic."""
import os
import shutil
import subprocess

import pytest

from unsuperviseddeephomographyral2018_b200 import build_ext


def _nvcc():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    return nvcc if os.path.exists(nvcc) else shutil.which("nvcc")


@pytest.mark.skipif(_nvcc() is None, reason="nvcc is not installed")
def test_no_serialised_wgmma(tmp_path):
    nvcc = _nvcc()
    procs = []
    for name in ("conv_x3.cu", "conv_tc.cu"):
        cmd = [nvcc] + build_ext.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build_ext.CSRC, name),
                                              "-o", str(tmp_path / (name[:-3] + ".o"))]
        procs.append((name, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    bad = []
    for name, p in procs:
        out, _ = p.communicate(timeout=900)
        assert p.returncode == 0, out
        assert "Compiling entry function" in out, "ptxas -v printed no kernel report for %s" % name
        for line in out.splitlines():
            if "(C7510)" in line or "(C7519)" in line:
                bad.append("%s: %s" % (name, line.strip()))
    assert not bad, "\n".join(bad)
