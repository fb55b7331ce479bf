"""Build libudh.so in-tree with nvcc for sm_90a (no torch in the link line: the library is a plain C ABI).

Concurrency: several ranks (torchrun) may import the package at once on a fresh clone.  The build runs under an exclusive
fcntl lock on `build/.lock`, compiles into a per-variant object directory, links to a temporary name and publishes the
library with an atomic rename — a concurrent importer either waits for the lock and then finds the library up to date, or
loads the previous complete file; it never sees a half-written one.

Variants: UDH_LIB_VARIANT=<name> builds libudh_<name>.so with the extra nvcc flags VARIANTS[name] into its own object
directory (for A/B experiments; the product is the default variant and the only one listed).
"""
import fcntl
import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")

VARIANTS = {"": []}


def variant():
    v = os.environ.get("UDH_LIB_VARIANT", "")
    if v not in VARIANTS:
        raise RuntimeError("unknown UDH_LIB_VARIANT %r (known: %s)" % (v, sorted(VARIANTS)))
    return v


def lib_path(v=None):
    v = variant() if v is None else v
    return os.path.join(HERE, "libudh%s.so" % ("_" + v if v else ""))


LIB = lib_path("")

NVCC_FLAGS = [
    "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
    "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr",
]


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def needs_build(v=None):
    lib = lib_path(v)
    if not os.path.exists(lib):
        return True
    t = os.path.getmtime(lib)
    deps = sources() + glob.glob(os.path.join(CSRC, "*.cuh")) + [os.path.join(HERE, "..", "include", "udh.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False, v=None):
    v = variant() if v is None else v
    lib = lib_path(v)
    if not force and not needs_build(v):
        return lib
    bdir = os.path.join(HERE, "build" + ("_" + v if v else ""))
    os.makedirs(bdir, exist_ok=True)
    with open(os.path.join(bdir, ".lock"), "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            if not force and not needs_build(v):        # another process built it while we waited for the lock
                return lib
            nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
            objs, procs = [], []
            for src in sources():
                obj = os.path.join(bdir, os.path.basename(src)[:-3] + ".o")
                objs.append(obj)
                cmd = [nvcc] + NVCC_FLAGS + VARIANTS[v] + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj]
                procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
            ok = True
            for src, p in procs:
                out, _ = p.communicate()
                if p.returncode != 0 or verbose:
                    sys.stderr.write("== %s\n%s\n" % (os.path.basename(src), out))
                ok = ok and p.returncode == 0
            if not ok:
                raise RuntimeError("nvcc failed building %s" % os.path.basename(lib))
            tmp = "%s.tmp.%d" % (lib, os.getpid())
            subprocess.check_call([nvcc, "-shared", "-o", tmp] + objs + ["-gencode", "arch=compute_90a,code=sm_90a"])
            os.replace(tmp, lib)                        # atomic publish
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)
    return lib


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
