"""Static audit of the programmatic-dependent-launch (PDL) chain (common.cuh: launch_chain, pdl_wait, pdl_trigger).

A kernel launched through launch_chain() may be scheduled while its predecessor in the stream is still running.  It is
correct only if (1) no path touches global memory before its griddepcontrol.wait and (2) every CTA reaches that wait, so
that completion is transitive along the chain.  In SASS griddepcontrol.wait is ACQBULK and griddepcontrol.launch_dependents
is PREEXIT.  This module finds the chained kernels in the sources, builds each compiled kernel's control-flow graph from its
SASS listing (cuobjdump -sass) and reports what is reachable from the entry without passing a wait."""
import os
import re
import shutil
import subprocess
from collections import Counter

# opcodes (the part before the first '.') that access global memory, or that touch memory outside the CTA and so must be
# justified when they run before the wait: UTMACCTL (tensor-map descriptor prefetch), the TMA and bulk-copy families, the
# generic LD / ST / ATOM (the address may be global) and the global loads, stores, atomics and reductions
GLOBAL_OPS = frozenset({
    "LDG", "STG", "ATOMG", "RED", "REDG", "LDGSTS", "UTMALDG", "UTMASTG", "UTMAREDG", "UTMAPF", "UTMACCTL", "UBLKCP",
    "UBLKRED", "UBLKPF", "LD", "ST", "ATOM",
})

_INSN = re.compile(r"/\*([0-9a-f]{4,})\*/\s+(@!?U?P(?:T|\d+)\s+)?([A-Z][A-Z0-9_.]*)\s*([^;]*);")
_FUNC = re.compile(r"Function : (\S+)")
_HEX = re.compile(r"0x([0-9a-f]+)")


class Insn:
    __slots__ = ("addr", "pred", "op", "args")

    def __init__(self, addr, pred, op, args):
        self.addr, self.pred, self.op, self.args = addr, pred, op, args

    @property
    def base(self):
        return self.op.split(".")[0]

    @property
    def predicated(self):
        # @PT is always true; any other guard may be false at run time
        return bool(self.pred) and self.pred not in ("@PT", "@UPT")

    def __repr__(self):
        return "/*%04x*/ %s%s %s" % (self.addr, (self.pred + " ") if self.pred else "", self.op, self.args)


def parse_sass(text):
    """cuobjdump -sass listing -> {mangled function name: [Insn, ...] in address order}."""
    funcs, cur = {}, None
    for line in text.splitlines():
        m = _FUNC.search(line)
        if m:
            cur = funcs.setdefault(m.group(1), [])
            continue
        if cur is None:
            continue
        m = _INSN.search(line)
        if m:
            pred = (m.group(2) or "").strip()
            cur.append(Insn(int(m.group(1), 16), pred, m.group(3), m.group(4).strip()))
    return funcs


def _target(insn):
    hx = _HEX.findall(insn.args)
    return int(hx[-1], 16) if hx else None


def successors(insns):
    """Control-flow successors of every instruction (indices).  Conservative: a predicated instruction may or may not
    take effect, a conditional branch both falls through and jumps, a call falls through and enters its target, and an
    indirect branch may go anywhere."""
    index = {x.addr: i for i, x in enumerate(insns)}
    succ = []
    for i, x in enumerate(insns):
        nxt = [i + 1] if i + 1 < len(insns) else []
        b = x.base
        if b in ("EXIT", "RET", "BPT", "KILL"):
            s = nxt if x.predicated else []
        elif b in ("BRX", "JMX"):
            s = list(range(len(insns)))
        elif b in ("BRA", "JMP", "CALL") or x.op == "WARPSYNC.COLLECTIVE":
            t = _target(x)
            s = [index[t]] if t in index else []
            unconditional = b in ("BRA", "JMP") and x.op == b and not x.predicated and "," not in x.args
            if not unconditional:
                s = s + nxt
        else:
            s = nxt
        succ.append(s)
    return succ


def is_wait(insn):
    return insn.base == "ACQBULK" and not insn.predicated


def pre_wait(insns):
    """Indices of the instructions reachable from the entry without passing an (unpredicated) ACQBULK.  ACQBULK dominates
    an instruction exactly when that instruction is not in this set."""
    if not insns:
        return set()
    succ = successors(insns)
    seen, stack = {0}, [0]
    while stack:
        i = stack.pop()
        if is_wait(insns[i]):
            continue
        for j in succ[i]:
            if j not in seen:
                seen.add(j)
                stack.append(j)
    return {i for i in seen if not is_wait(insns[i])}


def waits_first(insns):
    """True when the wait is in the entry basic block: straight-line code from the entry reaches an unpredicated ACQBULK
    with no branch, exit, call or branch target on the way, so every CTA waits before it does anything else."""
    targets = {_target(x) for x in insns if x.base in ("BRA", "JMP", "CALL", "BRX", "JMX")
               or x.op == "WARPSYNC.COLLECTIVE"}
    for k, x in enumerate(insns):
        if is_wait(x):
            return True
        if k > 0 and x.addr in targets:
            return False
        if x.base in ("BRA", "JMP", "CALL", "BRX", "JMX", "EXIT", "RET", "BPT", "KILL") or x.op == "WARPSYNC.COLLECTIVE":
            return False
    return False


class Verdict:
    """What one function does before its wait."""

    def __init__(self, insns):
        pre = pre_wait(insns)
        self.has_wait = any(is_wait(x) for x in insns)
        self.waits_first = waits_first(insns)
        self.pre_mem = Counter(insns[i].op for i in sorted(pre) if insns[i].base in GLOBAL_OPS)
        self.pre_exit = [insns[i] for i in sorted(pre) if insns[i].base == "EXIT"]
        self.pre_trigger = [insns[i] for i in sorted(pre) if insns[i].base == "PREEXIT"]
        self.has_trigger = any(x.base == "PREEXIT" for x in insns)

    def problems(self, allowed=None):
        """Violations of the chain contract; `allowed` = {opcode: count} of pre-wait accesses known to be safe."""
        out = []
        if not self.has_wait:
            out.append("no griddepcontrol.wait (ACQBULK)")
            return out
        if dict(self.pre_mem) != dict(allowed or {}):
            out.append("memory access before the wait: %s (allowed: %s)" % (dict(self.pre_mem), dict(allowed or {})))
        if self.pre_exit:
            out.append("EXIT reachable before the wait: %s" % self.pre_exit[0])
        if self.pre_trigger:
            out.append("launch_dependents (PREEXIT) reachable before the wait: %s" % self.pre_trigger[0])
        return out


# ---- names ------------------------------------------------------------------------------------------------------------

def base_of_mangled(name):
    """Unqualified function name of an Itanium-mangled symbol (_Z3foo..., _ZN3udh2tc3fooI...E...)."""
    if not name.startswith("_Z"):
        return name
    i = 2
    nested = name[i] == "N"
    if nested:
        i += 1
    last = None
    while i < len(name) and name[i].isdigit():
        j = i
        while name[j].isdigit():
            j += 1
        n = int(name[i:j])
        last = name[j:j + n]
        i = j + n
        if not nested:
            break
    return last


def short_name(name):
    """A demangled kernel name without return type, namespaces and parameters:
    'void udh::tc::foo<(int)1, (bool)0>(int, float*)' -> 'foo<(int)1, (bool)0>'."""
    name = name.replace("(anonymous namespace)::", "").replace("<unnamed>::", "")
    if name.startswith("void "):
        name = name[5:]
    depth = 0
    for i, c in enumerate(name):
        if c == "<":
            depth += 1
        elif c == ">":
            depth -= 1
        elif c == "(" and depth == 0:
            name = name[:i]
            break
    head, sep, args = name.partition("<")
    return head.split("::")[-1] + sep + args


def base_of_demangled(name):
    """Unqualified function name of a demangled kernel name ('void udh::tc::foo<1, 2>(int, float*)' -> 'foo')."""
    return short_name(name).split("<")[0]


# ---- what may run before the wait -------------------------------------------------------------------------------------
# (kernel, opcode, count per instantiation, why it is safe).  `kernel` is an fnmatch pattern over the short demangled name
# (short_name); an instantiation must show exactly the counts of the entries that match it.
PRE_WAIT_ALLOWED = [
    ("tc_gemm_kernel<*>", "UTMACCTL.PF", 2, "prefetch of the A and B tensor maps, __grid_constant__ parameters"),
    ("tc_conv_kernel<*, (bool)0, (int)?>", "UTMACCTL.PF", 3, "prefetch of the A128, Ahh and W tensor-map parameters"),
    ("tc_conv_kernel<*, (bool)1, (int)?>", "UTMACCTL.PF", 4, "the same and the TMA-store epilogue's output map"),
    ("tc_conv_x3_kernel<*>", "UTMACCTL.PF", 4, "prefetch of the A128, Ahh, W and output tensor-map parameters"),
    ("tc_wgrad_kernel<*>", "UTMACCTL.PF", 3, "prefetch of the X128, Xhh and G tensor-map parameters"),
    ("tc_wgrad_kernel<*>", "ST.E", 1, "the bf16 ones block in shared memory, through the re-aligned extern __shared__ pointer"),
    ("tc_wgrad64_kernel<*>", "UTMACCTL.PF", 3, "prefetch of the X128, Xhh and G136 tensor-map parameters"),
    ("tc_wgrad64_kernel<*>", "ST.E", 1, "the bf16 ones block in shared memory, through the re-aligned extern __shared__ pointer"),
    ("tc_wgrad_x3_kernel<*>", "UTMACCTL.PF", 3, "prefetch of the X128, Xhh and G tensor-map parameters"),
    ("tc_wgrad_x3_kernel<*>", "ST.E", 2, "fill_const_blocks: the constant limb blocks in shared memory (generic pointer)"),
    ("tc_wgrad64_x3_kernel<*>", "UTMACCTL.PF", 3, "prefetch of the X128, Xhh and G136 tensor-map parameters"),
    ("tc_wgrad64_x3_kernel<*>", "ST.E", 2, "fill_const_blocks: the constant limb blocks in shared memory (generic pointer)"),
    ("conv1_tc_wgrad_kernel", "UTMACCTL.PF", 1, "prefetch of the G tensor-map parameter"),
    ("conv1_tc_wgrad_kernel", "ST.E.128", 1, "zeroing the shared-memory A tile (generic pointer)"),
    ("conv1_x3_wgrad_kernel<*>", "UTMACCTL.PF", 1, "prefetch of the G tensor-map parameter"),
    ("conv1_x3_wgrad_kernel<*>", "ST.E.128", 1, "zeroing the shared-memory A tile (generic pointer)"),
    ("conv1_tc_fwd_kernel", "UTMACCTL.PF", 1, "prefetch of the output tensor-map parameter"),
    ("conv1_tc_fwd_kernel", "ST.E.128", 2, "zeroing the shared-memory A tile and storing the weight tile (generic pointer)"),
    ("conv1_tc_fwd_kernel", "LDG.E.CONSTANT", 8,
     "conv1_1's weights: PARAMETERS READ BEFORE THE WAIT, safe only while the launch before it waits at its top and no "
     "parameter writer runs in between (tests/test_gpu_pdl.py)"),
    ("conv1_x3_fwd_kernel<*>", "UTMACCTL.PF", 1, "prefetch of the output tensor-map parameter"),
    ("conv1_x3_fwd_kernel<*>", "ST.E.128", 3, "zeroing the shared-memory A tile and storing both weight limb tiles (generic pointer)"),
    ("conv1_x3_fwd_kernel<*>", "LDG.E.CONSTANT", 9,
     "conv1_1's weights and bias: PARAMETERS READ BEFORE THE WAIT, safe only while the launch before it waits at its top "
     "and no parameter writer runs in between (tests/test_gpu_pdl.py)"),
]

# kernels that read global memory before their wait (the allowlist's LDG entries): their predecessor on the stream decides
# whether what they read is final
PRE_WAIT_READERS = sorted({k.split("<")[0] for k, op, _, _ in PRE_WAIT_ALLOWED if op.startswith("LDG")})
# kernels that write the parameters (Adam's update; load_flat and checkpoint loads are copies, not kernels)
PARAM_WRITERS = ("adam_kernel",)


def pre_wait_order_problems(kernels, top_waiters, readers=PRE_WAIT_READERS, writers=PARAM_WRITERS):
    """The launch-order invariant of the pre-wait readers on a kernel trace [(stream, start, end, demangled name)]: each
    reader's predecessor on its stream waits in its first block (so the reader starts only after everything before that
    predecessor is complete) and writes no parameters, and no parameter writer on another stream runs between the
    predecessor's start and the reader's end.  Returns (readers checked, problems)."""
    by_stream = {}
    for k in sorted(kernels, key=lambda k: (k[1], k[2])):
        by_stream.setdefault(k[0], []).append(k)
    checked, out = 0, []
    for st, ks in by_stream.items():
        for i, (_, t0, t1, name) in enumerate(ks):
            if base_of_demangled(name) not in readers:
                continue
            checked += 1
            if i == 0:
                out.append("%s is the first kernel of stream %s: its predecessor is not in the trace" % (short_name(name), st))
                continue
            prev = ks[i - 1]
            pb = base_of_demangled(prev[3])
            if pb not in top_waiters or pb in writers:
                out.append("%s follows %s on stream %s, which %s" % (short_name(name), short_name(prev[3]), st,
                                                                     "writes the parameters" if pb in writers
                                                                     else "does not wait in its first block"))
            for o in kernels:
                if o[0] != st and base_of_demangled(o[3]) in writers and o[1] < t1 and o[2] > prev[1]:
                    out.append("%s on stream %s runs between %s and %s on stream %s" % (
                        short_name(o[3]), o[0], short_name(prev[3]), short_name(name), st))
    return checked, out


def overlapping_pairs(kernels, chained):
    """(consecutive chained pairs on one stream, how many of them overlap: the successor starts before the predecessor
    ends)."""
    by_stream = {}
    for k in sorted(kernels, key=lambda k: (k[1], k[2])):
        by_stream.setdefault(k[0], []).append(k)
    pairs = overlap = 0
    for ks in by_stream.values():
        for a, b in zip(ks, ks[1:]):
            if base_of_demangled(a[3]) in chained and base_of_demangled(b[3]) in chained:
                pairs += 1
                overlap += b[1] < a[2]
    return pairs, overlap


def allowed_for(short):
    """{opcode: count} that PRE_WAIT_ALLOWED grants the instantiation `short` (two entries for one opcode: error)."""
    import fnmatch
    out = {}
    for pat, op, n, _ in PRE_WAIT_ALLOWED:
        if fnmatch.fnmatchcase(short, pat):
            assert op not in out, "two allowlist entries grant %s to %s" % (op, short)
            out[op] = n
    return out


# ---- sources ----------------------------------------------------------------------------------------------------------

def _strip_comments(src):
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return re.sub(r"//[^\n]*", "", src)


def expand(csrc, name, seen=None):
    """Source text of `name` with its local ("...") includes inlined once, as the preprocessor would see them."""
    seen = set() if seen is None else seen
    if name in seen:
        return ""
    seen.add(name)
    path = os.path.join(csrc, name)
    if not os.path.exists(path):
        return ""
    out = []
    with open(path) as f:
        for line in f:
            m = re.match(r'\s*#include\s+"([^"]+)"', line)
            out.append(expand(csrc, m.group(1), seen) if m else line)
    return "".join(out)


def _first_arg(text, i):
    """The first argument of a call whose '(' is at text[i] (commas inside <> or () do not split it)."""
    depth, j = 0, i + 1
    while j < len(text):
        c = text[j]
        if c in "(<[":
            depth += 1
        elif c in ")>]":
            if depth == 0:
                break
            depth -= 1
        elif c == "," and depth == 0:
            break
        j += 1
    return text[i + 1:j].strip()


def _kernel_base(expr):
    expr = expr.lstrip("&").strip()
    m = re.match(r"[\w:]+", expr)
    return m.group(0).split("::")[-1] if m else expr


def _scan(text, pattern):
    """Kernel names at the call sites `pattern` (one group: the position of the opening bracket) in `text`.  A site that
    passes a variable (`launch_chain(kern, ...)`) resolves to the last `auto kern = <kernel>;` before it."""
    found = set()
    for m in re.finditer(pattern, text):
        first = _kernel_base(_first_arg(text, m.end() - 1)) if m.group(0).endswith("(") else _kernel_base(m.group(1))
        if re.fullmatch(r"[a-z_]\w*", first) and not first.endswith("_kernel"):
            decls = list(re.finditer(r"\b(?:auto|const auto)\s+%s\s*=\s*([^;]+);" % re.escape(first), text[:m.start()]))
            assert decls, "launch site passes %r but no `auto %s = <kernel>` precedes it" % (first, first)
            first = _kernel_base(decls[-1].group(1))
        found.add(first)
    return found


def chained_kernels(csrc, source):
    """Kernels that `source` (a .cu file, with its local includes) launches through launch_chain()."""
    text = _strip_comments(expand(csrc, source))
    text = re.sub(r"inline void launch_chain\(", "", text)          # the definition itself (common.cuh)
    return _scan(text, r"\blaunch_chain\(")


def plain_launched_kernels(csrc, source):
    """Kernels that `source` launches with the triple-chevron syntax."""
    text = _strip_comments(expand(csrc, source))
    return _scan(text, r"\b([\w:]+(?:<[^<>;]*>)?)\s*<<<")


# ---- toolchain ----------------------------------------------------------------------------------------------------------

def tool(name):
    p = os.path.join(os.path.dirname(os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")), name)
    return p if os.path.exists(p) else shutil.which(name)


def disassemble(path):
    p = subprocess.run([tool("cuobjdump"), "-sass", path], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                       timeout=600)
    assert p.returncode == 0, p.stdout[-4000:]
    return parse_sass(p.stdout)


def compile_objects(sources, flags, outdir, csrc):
    """nvcc -c every source (in parallel) with `flags`; returns {source: object path}."""
    procs = {}
    for s in sources:
        obj = os.path.join(outdir, os.path.splitext(os.path.basename(s))[0] + ".o")
        cmd = [tool("nvcc")] + list(flags) + ["-c", os.path.join(csrc, s), "-o", obj]
        procs[s] = (obj, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    out = {}
    for s, (obj, p) in procs.items():
        log, _ = p.communicate(timeout=1200)
        assert p.returncode == 0, "%s failed to compile:\n%s" % (s, log[-4000:])
        out[s] = obj
    return out


def demangle(names):
    """{mangled: demangled} through cu++filt (falls back to the mangled names)."""
    names = list(names)
    f = tool("cu++filt")
    if not f or not names:
        return {n: n for n in names}
    p = subprocess.run([f], input="\n".join(names), stdout=subprocess.PIPE, text=True, timeout=60)
    lines = p.stdout.splitlines()
    return dict(zip(names, lines)) if len(lines) == len(names) else {n: n for n in names}
