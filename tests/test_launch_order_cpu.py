"""The library's launch-order contract, checked on the PTX of every source (cross-compiled for sm_90a, no GPU needed).

Every kernel is launched with programmatic dependent launch (launch_kc in csrc/icaf_internal.cuh) and lets its successor
start at once (griddepcontrol.launch_dependents), so a kernel may run while its predecessor still writes.  That is only
correct while every kernel executes griddepcontrol.wait before it touches memory another kernel may have produced, and
before it completes (a grid that ends early would let its own successor pass the wait ahead of the predecessor).  A kernel
that breaks the rule reads stale data only sometimes, which no single-launch test notices; so a must-analysis over each
entry's control-flow graph checks that an unpredicated wait dominates every global / generic memory instruction and every
ret / exit.  The same pass checks that no kernel has a floating-point atomic, whose sum would depend on the order the
atomics land: the bit-identity of graphed and eager steps, and of ranks, rests on that.
"""
import collections
import os
import re
import shutil
import subprocess

import pytest

from icafusion_b200 import build as B


def _nvcc():
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    return exe if os.path.exists(exe) else None


CUB_PREFIX = "_ZN3cub"        # cub's radix sort kernels (metrics.cu): cub launches them itself, without the PDL attribute

# (instruction, entries it is allowed in (None: any), why it may precede the wait)
EXEMPT = {
    "prefetch.tensormap": (None, "prefetches a __grid_constant__ tensor map from the kernel's own parameter space, which no "
                                 "other kernel writes"),
    "prefetch.global.L2": ("prefetch_l2_kernel", "warms L2 with the next layer's filters; a prefetch changes no value and "
                                                 "the kernel still waits before it completes"),
}

_FLOAT_TYPES = ("f16", "f16x2", "bf16", "bf16x2", "f32", "f64")
_NO_GLOBAL = (".param", ".shared", ".local", ".const")
_MEM_OPS = re.compile(r"(ld|ldu|st|atom|red|multimem|prefetch|prefetchu)$")
_ASYNC_OPS = re.compile(r"(cp\.async|cp\.reduce\.async)(\.|$)")


def parse_entries(ptx):
    """{name: [instruction, ...]} of every .entry of a PTX module, and the same of every .func with a body."""
    entries, funcs = {}, {}
    for m in re.finditer(r"^(?:\.visible\s+|\.weak\s+)?\.(entry|func)\s+(?:\([^)]*\)\s*)?(\w+)", ptx, re.M):
        start, semi = ptx.find("\n{", m.end()), ptx.find(";", m.end())
        if start < 0 or 0 <= semi < start:
            continue                                     # a prototype without a body
        ins, depth = [], 0
        for line in ptx[start + 1:].split("\n"):
            line = line.split("//")[0]
            depth += line.count("{") - line.count("}")         # inline asm adds scopes of its own
            if depth == 0:
                break
            for part in line.replace("{", ";").replace("}", ";").split(";"):
                part = part.strip()
                if part:
                    ins.append(part)
        (entries if m.group(1) == "entry" else funcs)[m.group(2)] = ins
    return entries, funcs


def _opcode(ins):
    m = re.match(r"^(@!?%\w+\s+)?([A-Za-z_][\w.:]*)", ins)
    return (m.group(1) is not None, m.group(2)) if m else (False, "")


def _touches_global(op):
    """True for an instruction that may read or write global memory: ld / st / atom / red / prefetch / multimem in the
    global or generic state space, and the async copies with a global operand."""
    root = op.split(".")[0]
    if _MEM_OPS.match(root):
        return not any(s in op for s in _NO_GLOBAL) or ".global" in op
    if _ASYNC_OPS.match(op):
        return ".global" in op
    return False


def _blocks(ins):
    """Basic blocks, split at labels and after every branch, ret, exit and trap: [(label, [instruction])], ENTRY first."""
    blocks, seen = [("ENTRY", [])], set()
    for i in ins:
        m = re.match(r"^(\$?\w+):$", i)
        if m:
            assert m.group(1) not in seen, f"label {m.group(1)} defined twice (scoped labels are not handled)"
            seen.add(m.group(1))
            blocks.append((m.group(1), []))
            continue
        blocks[-1][1].append(i)
        if _opcode(i)[1].split(".")[0] in ("bra", "ret", "exit", "trap"):
            blocks.append((f"<after {len(blocks)}>", []))
    return blocks


def analyse(name, ins):
    """[(kind, instruction)] of what breaks the wait-first rule in one entry, kind in {mem, exit}; and the exemptions used."""
    blocks = _blocks(ins)
    labels = [b for b, _ in blocks]
    succ = {}
    for k, (b, body) in enumerate(blocks):
        s, falls = [], True
        for i in body:
            pred, op = _opcode(i)
            assert not op.startswith("brx"), f"{name}: indirect branch not handled: {i}"
            if op.split(".")[0] == "bra":
                tgt = i.split()[-1]
                assert tgt in labels, f"{name}: branch to unknown label {tgt}"
                s.append(tgt)
                falls = falls and pred
            elif op in ("ret", "exit", "trap") and not pred:
                falls = False
        if falls and k + 1 < len(blocks):
            s.append(labels[k + 1])
        succ[b] = s
    live, todo = {"ENTRY"}, ["ENTRY"]                    # blocks reachable from the entry (nvcc leaves empty dead ones)
    while todo:
        for t in succ[todo.pop()]:
            if t not in live:
                live.add(t)
                todo.append(t)
    labels = [b for b in labels if b in live]
    preds = collections.defaultdict(list)
    for b in labels:
        for t in succ[b]:
            preds[t].append(b)

    def waits(i):
        pred, op = _opcode(i)
        return op == "griddepcontrol.wait" and not pred

    body_of = dict(blocks)
    out = {b: True for b in labels}                     # must-analysis: top everywhere but at the entry
    inw = {b: True for b in labels}
    changed = True
    while changed:
        changed = False
        for b in labels:
            w = False if b == "ENTRY" else all(out[p] for p in preds[b])
            inw[b] = w
            o = w or any(waits(i) for i in body_of[b])
            if o != out[b]:
                out[b], changed = o, True
    cvta_param = {i.split()[1].rstrip(",") for i in ins if _opcode(i)[1].startswith("cvta.param")}
    issues, used = [], []
    for b in labels:
        w = inw[b]
        for i in body_of[b]:
            if waits(i):
                w = True
            if w:
                continue
            pred, op = _opcode(i)
            if op in ("ret", "exit"):
                issues.append(("exit", i))
            elif _touches_global(op):
                ex = EXEMPT.get(op)
                if op == "prefetch.tensormap":
                    ok = re.search(r"\[(%\w+)\]", i) is not None and re.search(r"\[(%\w+)\]", i).group(1) in cvta_param
                else:
                    ok = ex is not None and ex[0] is not None and ex[0] in name
                if ok:
                    used.append(op)
                else:
                    issues.append(("mem", i))
    return issues, used


def float_atomics(ins):
    out = []
    for i in ins:
        _, op = _opcode(i)
        if re.match(r"(atom|red|multimem\.red|cp\.reduce\.async)(\.|$)", op) and any(p in _FLOAT_TYPES for p in op.split(".")):
            out.append(i)
    return out


def check_module(ptx):
    """{entry: [finding]} over one module (cub's kernels skipped), the library entry count and the exemptions used."""
    entries, funcs = parse_entries(ptx)
    found, used, n = {}, collections.Counter(), 0
    for name, ins in entries.items():
        if name.startswith(CUB_PREFIX):
            used[CUB_PREFIX] += 1
            continue
        n += 1
        issues, u = analyse(name, ins)
        used.update(u)
        issues += [("float atomic", i) for i in float_atomics(ins)]
        if issues:
            found[name] = issues
    for name, ins in funcs.items():                     # calls are not followed: no callee may touch global memory
        bad = [("mem in callee", i) for i in ins if _touches_global(_opcode(i)[1])] + [("float atomic", i) for i in float_atomics(ins)]
        if bad:
            found[name] = bad
    return found, n, used


# ------------------------------------------------------------------------------------------------ the library's PTX

@pytest.fixture(scope="module")
def library_ptx(tmp_path_factory):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not available")
    d = tmp_path_factory.mktemp("ptx")
    flags = [f for f in B.NVCC_FLAGS if not f.startswith("--use_fast_math") and f not in ("-Xcompiler", "-fPIC")]
    procs = []
    for s in B.SOURCES:
        out = d / (s[:-3] + ".ptx")
        cmd = [nvcc, *flags, "-ptx", os.path.join(B.CSRC, s), "-o", str(out)]
        procs.append((s, out, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    ptx = {}
    for s, out, p in procs:
        log, _ = p.communicate(timeout=900)
        assert p.returncode == 0, f"nvcc -ptx {s}:\n{log}"
        ptx[s] = out.read_text()
    return ptx


def test_every_kernel_waits_before_memory_and_has_no_float_atomics(library_ptx):
    found, used, n = {}, collections.Counter(), 0
    for s, ptx in library_ptx.items():
        f, k, u = check_module(ptx)
        found.update({f"{s}: {name}": v[:4] for name, v in f.items()})
        n += k
        used.update(u)
    assert n >= 100, f"only {n} library entries parsed: the PTX parser has stopped matching"
    assert not found, "\n".join(f"{name}: {v}" for name, v in found.items())
    # every exemption still applies somewhere, so that the table cannot outlive the code it excuses
    for key in list(EXEMPT) + [CUB_PREFIX]:
        assert used[key] > 0, f"exemption {key} no longer used: remove it"


# ------------------------------------------------------------------------------------------------ the analyser itself

_HEAD = """
.version 8.5
.target sm_90a
.address_size 64

.visible .entry k(
	.param .u64 k_param_0,
	.param .u32 k_param_1
)
{
	.reg .pred 	%p<3>;
	.reg .b32 	%r<9>;
	.reg .b64 	%rd<9>;
	.reg .f32 	%f<3>;
"""
_TAIL = "\n}\n"


def _issues(body):
    found, n, _ = check_module(_HEAD + body + _TAIL)
    assert n == 1
    return found.get("k", [])


GOOD = """
	ld.param.u64 	%rd1, [k_param_0];
	ld.param.u32 	%r1, [k_param_1];
	griddepcontrol.launch_dependents;
	mov.u32 	%r2, %tid.x;
	setp.ge.s32 	%p1, %r2, %r1;
	griddepcontrol.wait;
	@%p1 bra 	$L__BB0_2;
	cvta.to.global.u64 	%rd2, %rd1;
	ld.global.nc.f32 	%f1, [%rd2];
	atom.global.add.u32 	%r3, [%rd2+4], 1;
	st.global.f32 	[%rd2+8], %f1;
$L__BB0_2:
	ret;
"""


def test_analyser_passes_the_wait_first_form():
    assert _issues(GOOD) == []


def test_analyser_flags_a_load_before_the_wait():
    body = GOOD.replace("\tgriddepcontrol.wait;\n", "\tld.global.nc.f32 \t%f2, [%rd1];\n\tgriddepcontrol.wait;\n")
    assert _issues(body) == [("mem", "ld.global.nc.f32 \t%f2, [%rd1]")]
    body = GOOD.replace("\tgriddepcontrol.wait;\n", "\tld.f32 \t%f2, [%rd1];\n\tgriddepcontrol.wait;\n")   # generic
    assert _issues(body) == [("mem", "ld.f32 \t%f2, [%rd1]")]


def test_analyser_flags_a_branch_that_skips_the_wait():
    body = GOOD.replace("\tgriddepcontrol.wait;\n\t@%p1 bra \t$L__BB0_2;\n", "\t@%p1 bra \t$L__BB0_1;\n\tgriddepcontrol.wait;\n$L__BB0_1:\n")
    kinds = [k for k, _ in _issues(body)]
    assert kinds.count("mem") == 3 and kinds.count("exit") == 1, kinds


def test_analyser_flags_a_predicated_wait():
    body = GOOD.replace("\tgriddepcontrol.wait;\n", "\t@%p1 griddepcontrol.wait;\n")
    kinds = [k for k, _ in _issues(body)]
    assert kinds.count("mem") == 3 and kinds.count("exit") == 1, kinds


def test_analyser_flags_an_early_exit_before_the_wait():
    body = GOOD.replace("\tgriddepcontrol.wait;\n\t@%p1 bra \t$L__BB0_2;\n",
                        "\t@%p1 bra \t$L__BB0_3;\n\tgriddepcontrol.wait;\n\tbra.uni \t$L__BB0_4;\n$L__BB0_3:\n\texit;\n$L__BB0_4:\n")
    assert _issues(body) == [("exit", "exit")]


def test_analyser_ignores_parameter_and_shared_space_before_the_wait():
    body = GOOD.replace("\tgriddepcontrol.launch_dependents;\n", "\tgriddepcontrol.launch_dependents;\n\tst.shared.u32 \t[%r1], %r2;\n"
                        "\tld.shared.u32 \t%r4, [%r1];\n\tcvta.param.u64 \t%rd5, %rd1;\n\tprefetch.tensormap \t[%rd5];\n")
    assert _issues(body) == []
    body = GOOD.replace("\tgriddepcontrol.launch_dependents;\n", "\tgriddepcontrol.launch_dependents;\n\tprefetch.tensormap \t[%rd1];\n"
                        "\tprefetch.global.L2 \t[%rd1];\n")
    assert [k for k, _ in _issues(body)] == ["mem", "mem"]


@pytest.mark.parametrize("atom,flagged", [("atom.global.add.f32 \t%f2, [%rd2+4], %f1;", True),
                                          ("red.global.add.f32 \t[%rd2+4], %f1;", True),
                                          ("atom.global.add.noftz.f16x2 \t%r5, [%rd2+4], %r4;", True),
                                          ("red.global.add.f64 \t[%rd2+4], %fd1;", True),
                                          ("atom.global.max.s32 \t%r5, [%rd2+4], %r4;", False),
                                          ("atom.global.exch.b32 \t%r5, [%rd2+4], %r4;", False)])
def test_analyser_flags_float_atomics_only(atom, flagged):
    body = GOOD.replace("\tatom.global.add.u32 \t%r3, [%rd2+4], 1;\n", "\t" + atom + "\n")
    assert [k for k, _ in _issues(body)] == (["float atomic"] if flagged else [])
