"""The persistent decoder's energy loop keeps its operands in registers (no GPU needed: cuobjdump on the in-tree .so).

The decoder kernels run 512 threads at the 128-register cap.  Shared memory takes nearly all of L1, so a spilled value
lives in L2: a spill store of a tile that was just requested waits for that tile's data, and its reload costs an L2
round trip.  An energy loop that holds the next tile of P in registers spilled that buffer on every tile
(232-324 bytes of spill stores per kernel), which made each tile wait for HBM."""
import re

from test_sass_cpu import _body, sass  # noqa: F401  (module-scoped fixture of the same library)


def _loops_with_mma(body):
    """(first, last) addresses of every backward branch whose range contains an HMMA: the tile loops of the energies."""
    ins = []
    for line in body.splitlines():
        m = re.search(r"/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;", line)
        if m:
            ins.append((int(m.group(1), 16), m.group(2)))
    loops = []
    for addr, text in ins:
        m = re.match(r"(?:@!?U?P\w+\s+)?BRA(?:\.\w+)*\s+(?:`\()?\S*?0x([0-9a-f]+)", text)
        if m and int(m.group(1), 16) < addr:
            inside = [t for a, t in ins if int(m.group(1), 16) <= a <= addr]
            if any("HMMA" in t for t in inside) and len(inside) < 1000:      # the tile loop, not the loop over steps
                loops.append(inside)
    return loops


def test_persistent_decoder_energy_loop_has_no_local_memory_traffic(sass):  # noqa: F811
    for name, body in _body(sass, "dec_scan_kernel").items():
        loops = _loops_with_mma(body)
        assert loops, name
        for inside in loops:
            local = [t for t in inside if re.search(r"\b(LDL|STL)\b", t)]
            assert not local, (name, local)
