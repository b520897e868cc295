"""CPU test (no GPU) of the fused frontend kernels' machine code in the built library: fused_qkv_kernel<C> and
fused_ff_kernel<C, OP> keep their loops in registers (a spill would put local-memory traffic into every 16-row group),
take every B fragment from the staged weights with ldmatrix.x4 (LDSM) rather than with two 32-bit shared loads
per MMA, and read their rows from the per-warp stage that cp.async (LDGSTS) fills, with 64-bit shared loads."""
import re

from support import sass

KERNEL = re.compile(r"_ZN2bt(?:15fused_ff_kernelILi(32|64)ELb([01])EE|16fused_qkv_kernelILi(32|64)EE)")
# "@!PT" never executes: ptxas places such dummy shared loads next to LDGSTS
OPCODE = re.compile(r"/\*[0-9a-f]{4,}\*/\s+(@!?U?P[T0-9]+\s+)?([A-Z][A-Z0-9_.]*)")


def _opcodes(lib_built):
    """{kernel name: {opcode: count}} over the six fused instantiations, never-executed instructions left out."""
    ops, fn = {}, None
    for line in sass(lib_built).splitlines():
        if "Function :" in line:
            m = KERNEL.search(line)
            fn = (f"fused_ff_kernel<{m.group(1)}, {'true' if m.group(2) == '1' else 'false'}>" if m.group(1)
                  else f"fused_qkv_kernel<{m.group(3)}>") if m else None
            if fn:
                ops[fn] = {}
        elif fn:
            m = OPCODE.search(line)
            if m and m.group(1) != "@!PT ":
                ops[fn][m.group(2)] = ops[fn].get(m.group(2), 0) + 1
    assert len(ops) == 6, f"expected the six fused instantiations, found {sorted(ops)}"
    return ops


def test_fused_kernels_have_no_local_memory_access(lib_built):
    local = {fn: {op: n for op, n in c.items() if op.split(".")[0] in ("LDL", "STL")} for fn, c in _opcodes(lib_built).items()}
    assert not any(local.values()), f"local-memory accesses (spills): {local}"


def test_fused_kernels_take_b_fragments_from_ldmatrix(lib_built):
    """Every shared-memory load is an LDSM (weights, one per two MMAs) or a 64-bit LDS (stage rows); no 32-bit LDS
    feeds an HMMA."""
    for fn, c in _opcodes(lib_built).items():
        lds = {op: n for op, n in c.items() if op.startswith("LDS")}
        print(f"{fn}: {lds}, HMMA {c.get('HMMA.16816.F32', 0)}, LDGSTS {c.get('LDGSTS.E.BYPASS.128', 0)}")
        assert set(lds) == {"LDSM.16.M88.4", "LDS.64"}, f"{fn}: shared loads {lds}"
        assert 2 * lds["LDSM.16.M88.4"] == c["HMMA.16816.F32"], f"{fn}: {lds['LDSM.16.M88.4']} LDSM for {c['HMMA.16816.F32']} HMMA"
        assert c.get("LDGSTS.E.BYPASS.128", 0) > 0, f"{fn}: rows not staged by cp.async"
