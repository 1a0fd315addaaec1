"""CPU: the kernels csrc/ launches with programmatic dependent launch (r3g_launch_pdl) are exactly the consumers the GPU
chain tests cover (tests/test_gpu_pdl_chains.py: CONSUMERS), each calls pdl_wait(), and the chain table meets its
coverage rules.  A new PDL launch without a chain test fails here, before it reaches a GPU."""
import os
import re

import test_gpu_pdl_chains as chains

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "3d-re-gen_b200", "csrc")


def _sources():
    return {f: open(os.path.join(CSRC, f)).read() for f in sorted(os.listdir(CSRC)) if f.endswith(".cu")}


def pdl_launched_kernels(src):
    """Kernel instantiations passed to r3g_launch_pdl in one translation unit: a kernel named directly, a template
    kernel over the enclosing function's template parameter (every explicit instantiation of that function), or the
    parameter of a `go` / `args` lambda (every kernel the lambda is called with)."""
    found = set()
    for m in re.finditer(r"r3g_launch_pdl\(\s*ctx\s*,\s*([\w<>]+)\s*,", src):
        arg, pos = m.group(1), m.start()
        lam = list(re.finditer(r"auto\s+(\w+)\s*=\s*\[&\]\s*\(\s*auto\s+" + re.escape(arg) + r"\s*\)", src[:pos]))
        if lam:
            name = lam[-1].group(1)
            end = src.find('extern "C"', pos)
            calls = re.findall(r"\b" + name + r"\(\s*(\w+(?:<\d+>)?)\s*\)", src[pos:end if end >= 0 else len(src)])
            assert calls, f"lambda {name} is never called"
            found.update(calls)
            continue
        t = re.fullmatch(r"(\w+)<([A-Za-z_]\w*)>", arg)
        if t:
            fn = list(re.finditer(r"template\s*<int\s+" + t.group(2) + r">\s*\w+\s+(\w+)\(", src[:pos]))
            assert fn, f"no enclosing template function for {arg}"
            inst = set(re.findall(r"\b" + fn[-1].group(1) + r"<(\d+)>\(", src))
            assert inst, f"{fn[-1].group(1)} is never instantiated"
            found.update(f"{t.group(1)}<{n}>" for n in inst)
            continue
        found.add(arg)
    return found


def kernel_body(src, name):
    m = re.search(r"__global__[^;{]*?\b" + re.escape(name) + r"\s*\(", src)
    if m is None:
        return None
    i = src.index("{", m.end())
    depth = 0
    for j in range(i, len(src)):
        depth += {"{": 1, "}": -1}.get(src[j], 0)
        if depth == 0:
            return src[i:j + 1]
    raise AssertionError(f"unbalanced braces in {name}")


def test_pdl_launches_are_the_chain_consumers():
    launched = set()
    for src in _sources().values():
        launched |= pdl_launched_kernels(src)
    assert launched == set(chains.CONSUMERS), (f"launched with PDL but not in CONSUMERS: {sorted(launched - set(chains.CONSUMERS))}; "
                                               f"in CONSUMERS but not launched: {sorted(set(chains.CONSUMERS) - launched)}")


def test_every_pdl_kernel_waits():
    srcs = _sources()
    for k in chains.CONSUMERS:
        base = k.split("<")[0]
        bodies = [b for b in (kernel_body(s, base) for s in srcs.values()) if b is not None]
        assert len(bodies) == 1, f"{base}: {len(bodies)} definitions"
        assert "pdl_wait();" in bodies[0], f"{base} is launched with PDL but never calls pdl_wait()"


def test_early_triggering_kernels_are_the_listed_ones():
    srcs = _sources()
    entry_of = {"kv_fill_kernel": "kv_fill", **{k: v for k, v in chains.ENTRY.items() if k != "kv_fill_kernel"}}
    triggering = {entry_of[k.split("<")[0]] for k in chains.CONSUMERS
                  if "pdl_trigger();" in next(b for b in (kernel_body(s, k.split("<")[0]) for s in srcs.values()) if b)}
    assert triggering == set(chains.EARLY_TRIGGERING)


def test_chain_table_covers_every_consumer_producer_operand_and_overwrite():
    specs = chains.CHAINS
    assert len({s.name for s in specs}) == len(specs)
    covered = {k for s in specs for k in s.consumers}
    assert covered == set(chains.CONSUMERS), sorted(set(chains.CONSUMERS) - covered)
    producers = {s.producer for s in specs} | {"kv_fill" for s in specs if "kv_fill_kernel" in s.consumers}
    assert set(chains.EARLY_TRIGGERING) <= producers, sorted(set(chains.EARLY_TRIGGERING) - producers)
    for entry, operands in chains.ACTIVATION_OPERANDS.items():
        read = {r for s in specs if s.entry == entry and s.producer in chains.EARLY_TRIGGERING for r in s.reads}
        assert operands <= read, f"{entry}: no early-triggering producer writes {sorted(operands - read)}"
        assert any(s.war for s in specs if s.entry == entry), f"{entry}: no chain writes over the producer's input"
    for s in specs:
        assert all(chains.ENTRY[k.split("<")[0]] == s.entry for k in s.consumers), s.name
    assert any(s.side_stream for s in specs)
    assert sum(s.source is not None for s in specs) >= 16
