"""Static checks on the resident kernel's lookahead passes (staged_look_pass, no GPU): the eval-with-lookahead loop and
the double-bind loop stage their tables through shared memory with bulk copies, keep to registers (no local memory, no
generic accesses) and leave the kernels at 128 registers, so two blocks still fit on an SM. Reads resident.o /
resident.ptxas.log that `make -C jolt_b200/csrc` leaves in-tree; skipped before a build."""
import re
import shutil
import subprocess

import pytest

from test_build_artifacts_staged import CSRC, D2, _loops, _need


def _staged_loops(order):
    obj = _need(CSRC / "resident.o")
    cuobjdump = shutil.which("cuobjdump")
    if cuobjdump is None:
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", "-fun", D2[order], str(obj)], capture_output=True, text=True, timeout=600).stdout
    return [c for c in _loops(sass) if any(k.startswith("SYNCS.PHASECHK") for k in c) and any(k.startswith("UBLKCP") for k in c)
            and not any(k.startswith("REDUX") for k in c)]


def test_look_pass_functions_fit_the_kernel_budget():
    log = _need(CSRC / "resident.ptxas.log").read_text()
    assert "staged_look_pass" in log
    regs = {}
    cur = None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", line)
        if m:
            cur = m.group(1)
        m = re.search(r"Used (\d+) registers", line)
        if m and cur in D2.values():
            regs[cur] = int(m.group(1))
    assert set(regs) == set(D2.values()) and all(r <= 128 for r in regs.values()), regs


@pytest.mark.parametrize("order", sorted(D2))
def test_look_loops_stage_through_shared_memory(order):
    loops = _staged_loops(order)
    # eval + lookahead: the eight products' operands come straight out of the stage (many 128-bit shared loads);
    # double bind: every thread stores its T2 entry (STG.E.128) and exchanges it through shared memory (STS / LDS)
    look = [c for c in loops if c["LDS.128"] >= 32]
    bind2 = [c for c in loops if c["STS"] >= 8 and any(k.startswith("STG.E.128") for k in c)]
    assert look and bind2, loops
    for c in look + bind2:
        assert not any(k.startswith(("LDL", "STL")) for k in c), c         # no local memory
        assert not any(k.startswith(("LD.E", "ST.E")) for k in c), c       # no generic loads / stores
        assert c["LDS.128"] >= 4 and any(k.startswith("UBLKCP") for k in c), c
        assert sum(v for k, v in c.items() if k.startswith("IMAD.WIDE")) >= 60, c
