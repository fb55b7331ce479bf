"""The PDL chain audit (tests/_pdl_audit.py) on its own: hand-written SASS listings with a known answer (a branch around the
wait, an EXIT before it, a predicated load before it, a loop back-edge, a clean kernel), the source scan on a toy source
tree, and two tiny kernels compiled here, one that waits before its load and one that loads first.  An analyser that
found nothing would fail these."""
import textwrap

import pytest

import _pdl_audit as A


def listing(name, body):
    """A cuobjdump-style listing of one function from 'OPCODE operands' lines (addresses assigned 0x10 apart)."""
    lines = ["\t\tFunction : %s" % name, "\t.headerflags\t@\"EF_CUDA_SM90\""]
    for i, ins in enumerate(l.strip() for l in body.strip().splitlines()):
        lines.append("        /*%04x*/                   %s ;   /* 0x000000000000 */" % (16 * i, ins))
        lines.append("                                                            /* 0x000fe20000000000 */")
    return "\n".join(lines) + "\n"


def verdict(body, name="_Z1kPf"):
    funcs = A.parse_sass(listing(name, body))
    return A.Verdict(funcs[name])


CLEAN = """
    LDC R1, c[0x0][0x28]
    ACQBULK
    S2R R0, SR_TID.X
    PREEXIT
    LDG.E R2, desc[UR4][R2.64]
    STG.E desc[UR4][R4.64], R2
    EXIT
    BRA 0x70
"""


def test_clean_kernel():
    v = verdict(CLEAN)
    assert v.has_wait and v.waits_first and v.has_trigger
    assert v.problems() == []


def test_branch_around_the_wait():
    # @P0 jumps over the wait straight to the load
    v = verdict("""
        S2R R0, SR_TID.X
        ISETP.NE.AND P0, PT, R0, RZ, PT
        @P0 BRA 0x40
        ACQBULK
        LDG.E R2, desc[UR4][R2.64]
        PREEXIT
        EXIT
    """)
    assert v.has_wait and not v.waits_first
    assert v.pre_mem == {"LDG.E": 1}
    assert v.pre_trigger and "PREEXIT" in repr(v.pre_trigger[0])
    assert any("before the wait" in p for p in v.problems())


def test_exit_before_the_wait():
    # CTAs with no work leave before waiting: their successor would not inherit completion from them
    v = verdict("""
        S2R R0, SR_CTAID.X
        ISETP.GE.AND P0, PT, R0, 0x4, PT
        @P0 EXIT
        ACQBULK
        PREEXIT
        STG.E desc[UR4][R4.64], R2
        EXIT
    """)
    assert v.pre_mem == {}
    assert len(v.pre_exit) == 1 and v.pre_exit[0].addr == 0x20
    assert any("EXIT reachable" in p for p in v.problems())


def test_predicated_load_before_the_wait_counts():
    v = verdict("""
        ISETP.NE.AND P0, PT, R0, RZ, PT
        @P0 LDG.E.CONSTANT R3, desc[UR4][R2.64]
        ACQBULK
        PREEXIT
        EXIT
    """)
    assert v.pre_mem == {"LDG.E.CONSTANT": 1}
    assert v.problems({"LDG.E.CONSTANT": 1}) == []
    assert v.problems({"LDG.E.CONSTANT": 2})                 # a count that differs from the allowance fails


def test_predicated_wait_is_no_wait():
    v = verdict("""
        @P0 ACQBULK
        LDG.E R2, desc[UR4][R2.64]
        EXIT
    """)
    assert not v.has_wait
    assert v.problems() == ["no griddepcontrol.wait (ACQBULK)"]


def test_loop_back_edge_before_the_wait():
    # a shared-memory fill loop ahead of the wait, with a global load at its bottom: the back-edge keeps it pre-wait, and
    # the loads after the wait (reached through the loop exit) stay post-wait
    v = verdict("""
        MOV R0, RZ
        STS [R0], RZ
        LD.E R5, [R6.64]
        IADD3 R0, R0, 0x10, RZ
        ISETP.LT.AND P0, PT, R0, 0x100, PT
        @P0 BRA 0x10
        ACQBULK
        PREEXIT
        LDG.E R2, desc[UR4][R2.64]
        EXIT
    """)
    assert not v.waits_first
    assert v.pre_mem == {"LD.E": 1}
    assert not v.pre_exit and not v.pre_trigger


def test_loop_around_the_wait_back_to_the_entry():
    # a back-edge from after the wait to before it re-enters pre-wait code, which is fine: the wait was passed once
    v = verdict("""
        ACQBULK
        PREEXIT
        LDG.E R2, desc[UR4][R2.64]
        @P0 BRA 0x20
        EXIT
    """)
    assert v.waits_first and v.problems() == []


def test_call_and_shared_ops_and_unconditional_branch():
    # an unconditional BRA does not fall through; a call enters its subroutine; LDS / STS / ATOMS are not global
    v = verdict("""
        STS [R0], RZ
        ATOMS.ADD RZ, [R0], R1
        BRA 0x40
        LDG.E R2, desc[UR4][R2.64]
        CALL.REL.NOINC 0x80
        ACQBULK
        PREEXIT
        EXIT
        STG.E desc[UR4][R4.64], R2
        RET.REL.NODEC R20 0x0
    """)
    assert v.pre_mem == {"STG.E": 1}                         # the subroutine's store, not the skipped load
    assert not v.waits_first


def test_names():
    assert A.base_of_mangled("_ZN3udh2tc17tc_conv_x3_kernelILi64ELi1ELi2ELi0ELi0ELi0ELi0EEEvv") == "tc_conv_x3_kernel"
    assert A.base_of_mangled("_ZN3udh44_GLOBAL__N__5f015734_11_cnn_simt_cu_3bfcce3612sgemm_kernelEPKf") == "sgemm_kernel"
    assert A.base_of_mangled("_Z10bad_kernelPKfPf") == "bad_kernel"
    assert A.base_of_demangled("void udh::tc::tc_conv_x3_kernel<64, 1, 2, 0, 0, 0, 1>(CUtensorMap_st, int)") == "tc_conv_x3_kernel"
    assert A.base_of_demangled("void udh::(anonymous namespace)::pad_cast_x3_kernel<0>(float const*)") == "pad_cast_x3_kernel"
    assert A.base_of_demangled("udh::adam_kernel(float4*)") == "adam_kernel"


def test_source_scan(tmp_path):
    (tmp_path / "k.cuh").write_text(textwrap.dedent("""
        template <int N> __global__ void hdr_kernel(float* p) { pdl_wait(); pdl_trigger(); }
        template <int N> int launch_hdr(float* p, cudaStream_t st) {
          auto kern = hdr_kernel<N>;
          launch_chain(kern, dim3(1), dim3(32), 0, st, p);    // resolved through `auto kern`
          return 0;
        }
    """))
    (tmp_path / "a.cu").write_text(textwrap.dedent("""
        #include "k.cuh"
        // launch_chain(commented_kernel, ...) is not a launch
        int f(float* p, cudaStream_t st) {
          launch_chain(udh::one_kernel<3, true>, dim3(1), dim3(32), 0, st, p);
          udh::launch_chain(two_kernel, dim3(1), dim3(32), 0, st, p);
          plain_kernel<<<1, 32, 0, st>>>(p);
          tmpl_kernel<kGrad><<<1, 32>>>(p);
          return launch_hdr<1>(p, st);
        }
    """))
    assert A.chained_kernels(str(tmp_path), "a.cu") == {"one_kernel", "two_kernel", "hdr_kernel"}
    assert A.plain_launched_kernels(str(tmp_path), "a.cu") == {"plain_kernel", "tmpl_kernel"}


TINY = r"""
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__global__ void good_kernel(const float* __restrict__ x, float* __restrict__ y, int n) {
  pdl_wait(); pdl_trigger();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) y[i] = 2.f * x[i];
}
__global__ void bad_kernel(const float* __restrict__ x, float* __restrict__ y, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const float v = i < n ? __ldg(x + i) : 0.f;     // read before the wait: may see the predecessor's half-written output
  pdl_wait(); pdl_trigger();
  if (i < n) y[i] = 2.f * v;
}
__global__ void early_exit_kernel(float* __restrict__ y, int n) {
  if ((int)blockIdx.x * (int)blockDim.x >= n) return;    // CTAs without items leave before the wait
  pdl_wait(); pdl_trigger();
  y[blockIdx.x * blockDim.x + threadIdx.x] = 1.f;
}
"""


@pytest.mark.skipif(A.tool("nvcc") is None or A.tool("cuobjdump") is None, reason="the CUDA toolkit is not installed")
def test_compiled_good_and_bad_kernels(tmp_path):
    from unsuperviseddeephomographyral2018_b200 import build_ext
    (tmp_path / "tiny.cu").write_text(TINY)
    objs = A.compile_objects(["tiny.cu"], build_ext.NVCC_FLAGS, str(tmp_path), str(tmp_path))
    funcs = {A.base_of_mangled(k): v for k, v in A.disassemble(objs["tiny.cu"]).items()}
    good, bad, early = (A.Verdict(funcs[k]) for k in ("good_kernel", "bad_kernel", "early_exit_kernel"))
    print("good:", good.problems(), "\nbad:", bad.problems(), "\nearly exit:", early.problems())
    assert good.problems() == [] and good.waits_first
    assert any(op.startswith("LDG") for op in bad.pre_mem), bad.pre_mem
    assert bad.problems()
    assert early.pre_exit and early.problems()


def test_pre_wait_order_on_a_trace():
    """The launch-order check of tests/test_gpu_pdl.py on hand-made traces: the forward's order, conv1 launched before the
    weight pack, conv1 right after Adam, and Adam on a second stream across conv1's start."""
    top = {"pack_all_weights_x3_kernel", "adam_kernel", "pad_cast_x3_kernel"}
    pack = "void udh::(anonymous namespace)::pack_all_weights_x3_kernel(udh::PackTableX3)"
    conv1 = "void udh::tc::conv1_x3_fwd_kernel<1>(CUtensorMap_st, udh::tc::Conv1Geom, float const*)"
    adam = "udh::adam_kernel(float4*, float4*)"
    conv = "void udh::tc::tc_conv_x3_kernel<64, 1, 2, 1, 1, 1, 1>(CUtensorMap_st)"
    good = [(7, 0, 10, adam), (7, 11, 20, pack), (7, 19, 40, conv1), (7, 39, 60, conv)]
    assert A.pre_wait_order_problems(good, top) == (1, [])
    swapped = [(7, 0, 10, adam), (7, 11, 30, conv1), (7, 31, 40, pack), (7, 41, 60, conv)]
    n, p = A.pre_wait_order_problems(swapped, top)
    assert n == 1 and len(p) == 1 and "conv1_x3_fwd_kernel<1> follows adam_kernel" in p[0] and "writes the parameters" in p[0]
    after_conv = [(7, 0, 10, conv), (7, 9, 30, conv1)]
    assert "does not wait in its first block" in A.pre_wait_order_problems(after_conv, top)[1][0]
    side = good + [(9, 15, 25, adam)]
    n, p = A.pre_wait_order_problems(side, top)
    assert len(p) == 1 and "adam_kernel on stream 9 runs between" in p[0]
    assert "first kernel of stream" in A.pre_wait_order_problems([(7, 0, 1, conv1)], top)[1][0]
    chained = {"pack_all_weights_x3_kernel", "conv1_x3_fwd_kernel", "tc_conv_x3_kernel", "adam_kernel"}
    assert A.overlapping_pairs(good, chained) == (3, 2)
