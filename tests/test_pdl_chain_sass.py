"""The programmatic-dependent-launch chain, checked on the SASS the library ships (DESIGN.md section 2, "The PDL chain").

launch_chain() (common.cuh) lets a kernel's CTAs start while its predecessor in the stream still runs.  That is correct only
if every chained kernel (1) touches no global memory before griddepcontrol.wait (ACQBULK) on any path and (2) lets no CTA
leave before the wait, so that completion is transitive along the chain.  This compiles every source that chains kernels
exactly as the library build does, finds the chained kernels in the sources, and checks each compiled instantiation:
  (a) it contains ACQBULK;
  (b) ACQBULK dominates every global-memory instruction, except the allowlisted ones (_pdl_audit.PRE_WAIT_ALLOWED), whose
      counts must match exactly;
  (c) no EXIT is reachable before ACQBULK;
  (d) launch_dependents (PREEXIT) is not reachable before ACQBULK.
And in reverse: every function that waits is chained, or listed in WAITS_UNCHAINED with the reason."""
import fnmatch
import os

import pytest

import _pdl_audit as A
from unsuperviseddeephomographyral2018_b200 import build_ext

# source -> the kernels it launches through launch_chain() (with the headers it includes)
CHAINED = {
    "cnn_simt.cu": {"sgemm_kernel", "bias_act_dropout_kernel", "drop_relu_bwd_kernel", "colsum_kernel"},
    "conv_tc.cu": {"pack_all_weights_kernel", "pad_cast_kernel", "pool_fwd_bf16_kernel", "pool_bwd_bf16_kernel",
                   "cast_bf16_kernel", "tc_conv_kernel", "tc_wgrad_kernel", "tc_wgrad64_kernel", "tc_gemm_kernel",
                   "conv1_tc_fwd_kernel", "conv1_tc_wgrad_kernel"},
    "conv_x3.cu": {"pack_all_weights_x3_kernel", "pad_cast_x3_kernel", "cast_x3_kernel", "cast_planes_x3_kernel",
                   "pool_fwd_x3_kernel", "pool_bwd_x3_kernel", "tc_conv_x3_kernel", "tc_wgrad_x3_kernel",
                   "tc_wgrad64_x3_kernel", "tc_gemm_kernel", "conv1_x3_fwd_kernel", "conv1_x3_wgrad_kernel"},
    "dlt.cu": {"dlt_fwd_kernel"},
    "misc.cu": {"h4p_loss_kernel", "adam_kernel", "slab_reduce_kernel"},
    "warp.cu": {"warp_loss_fwd_kernel", "ssim_kernel", "photo_finalize_kernel"},
}
# (source, kernel) that contain a wait but are not chained from that source's object, and why
WAITS_UNCHAINED = {
    ("conv_x3.cu", "conv1_tc_fwd_kernel"): "compiled in through conv1_x3_kernels.cuh; launched from conv_tc.cu only",
    ("conv_x3.cu", "conv1_tc_wgrad_kernel"): "compiled in through conv1_x3_kernels.cuh; launched from conv_tc.cu only",
}
# chained instantiations per source as built today (nvcc 12.9, sm_90a): 57, plus the two WAITS_UNCHAINED copies = 59
# functions that wait
COUNTS = {"cnn_simt.cu": 4, "conv_tc.cu": 23, "conv_x3.cu": 20, "dlt.cu": 1, "misc.cu": 3, "warp.cu": 6}

needs_toolkit = pytest.mark.skipif(A.tool("nvcc") is None or A.tool("cuobjdump") is None,
                                   reason="the CUDA toolkit is not installed")


def chaining_sources():
    """Every .cu file of the library whose translation unit contains a launch_chain() call."""
    return sorted(os.path.basename(s) for s in build_ext.sources() if A.chained_kernels(build_ext.CSRC, os.path.basename(s)))


def test_chained_table_matches_the_sources():
    found = {s: A.chained_kernels(build_ext.CSRC, s) for s in chaining_sources()}
    assert found == CHAINED, "launch_chain() sites changed: update CHAINED (and check the new kernels' waits)\n%s" % (
        "\n".join("%s: +%s -%s" % (s, sorted(found.get(s, set()) - CHAINED.get(s, set())),
                                    sorted(CHAINED.get(s, set()) - found.get(s, set())))
                  for s in sorted(set(found) | set(CHAINED)) if found.get(s) != CHAINED.get(s)))


@pytest.fixture(scope="module")
def sass(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("pdl_sass"))
    objs = A.compile_objects(sorted(CHAINED), build_ext.NVCC_FLAGS, out, build_ext.CSRC)
    funcs = {s: A.disassemble(o) for s, o in objs.items()}
    names = A.demangle([n for f in funcs.values() for n in f])
    return {s: {n: (A.short_name(names[n]), insns) for n, insns in f.items()} for s, f in funcs.items()}


@needs_toolkit
def test_every_chained_kernel_waits_before_touching_global_memory(sass):
    bad, counts, used = [], {}, set()
    for src in sorted(CHAINED):
        seen = set()
        for mangled, (short, insns) in sorted(sass[src].items(), key=lambda kv: kv[1][0]):
            base = A.base_of_mangled(mangled)
            if base not in CHAINED[src]:
                continue
            seen.add(base)
            allowed = A.allowed_for(short)
            used.update((pat, op) for pat, op, _, _ in A.PRE_WAIT_ALLOWED if fnmatch.fnmatchcase(short, pat))
            v = A.Verdict(insns)
            problems = v.problems(allowed)
            counts[src] = counts.get(src, 0) + 1
            print("%-11s %-78s %s%s" % (src, short[:78], "OK" if not problems else "FAIL",
                                        (" (before the wait: %s)" % dict(v.pre_mem)) if v.pre_mem else ""))
            bad += ["%s: %s: %s" % (src, short, p) for p in problems]
        missing = CHAINED[src] - seen
        assert not missing, "%s: chained kernels with no compiled instantiation: %s" % (src, sorted(missing))
    stale = {(pat, op) for pat, op, _, _ in A.PRE_WAIT_ALLOWED} - used
    assert not bad, "\n".join(bad)
    assert not stale, "allowlist entries that no chained instantiation uses: %s" % sorted(stale)
    assert counts == COUNTS, counts


@needs_toolkit
def test_every_waiting_kernel_is_chained(sass):
    """The reverse: a function with griddepcontrol.wait that is not launched through launch_chain() is listed with its
    reason (a wait in a plain launch is a no-op, which is harmless but says the kernel was meant to be chained)."""
    plain = {s: A.plain_launched_kernels(build_ext.CSRC, s) for s in CHAINED}
    found = {}
    for src, funcs in sass.items():
        for mangled, (short, insns) in funcs.items():
            base = A.base_of_mangled(mangled)
            if any(A.is_wait(x) for x in insns) and base not in CHAINED[src]:
                found[(src, base)] = "launched with <<<>>>" if base in plain[src] else "not launched from this source"
    assert set(found) == set(WAITS_UNCHAINED), found
    for k in WAITS_UNCHAINED:
        assert k[1] not in plain[k[0]], "%s waits and is launched with <<<>>> from %s" % (k[1], k[0])


@needs_toolkit
def test_pre_wait_readers_and_their_predecessors(sass):
    """The kernels that read parameters before their wait are exactly the conv1_1 forwards, and the weight packs that the
    forward launches right before them wait in their first instruction block (tests/test_gpu_pdl.py checks the launch
    order on the device)."""
    assert A.PRE_WAIT_READERS == ["conv1_tc_fwd_kernel", "conv1_x3_fwd_kernel"]
    top = {}
    for src, funcs in sass.items():
        for mangled, (short, insns) in funcs.items():
            base = A.base_of_mangled(mangled)
            if base in CHAINED[src]:
                top[base] = top.get(base, True) and A.waits_first(insns)
    assert top["pack_all_weights_kernel"] and top["pack_all_weights_x3_kernel"]
    print("chained kernels that wait in their first block:", sorted(k for k, v in top.items() if v))
