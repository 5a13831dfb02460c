"""Static checks on the resident kernel's staged passes (no GPU): they keep two blocks per SM and their hot loop is
what the design says - bulk copies into shared memory, shared-memory loads, no local memory, no generic accesses.
Reads resident.o / resident.ptxas.log that `make -C jolt_b200/csrc` leaves in-tree; skipped before a build."""
import collections
import pathlib
import re
import shutil
import subprocess

import pytest

from test_build_artifacts import ptxas_entries

CSRC = pathlib.Path(__file__).resolve().parents[1] / "jolt_b200" / "csrc"
D2 = {"h2l": "_ZN2jb22resident_rounds_kernelILi2ELi1ELi0EEEvNS_7ResArgsE",
      "l2h": "_ZN2jb22resident_rounds_kernelILi2ELi1ELi1EEEvNS_7ResArgsE"}


def _need(path):
    if not path.exists():
        pytest.skip("no build in this tree yet (python -c 'import __graft_entry__ as g; g.build()')")
    return path


def test_resident_kernels_keep_128_registers_and_their_static_shared_memory():
    log = _need(CSRC / "resident.ptxas.log")
    ents = {k: v for k, v in ptxas_entries(log).items() if "resident_rounds_kernel" in k}
    assert len(ents) >= 10
    assert all(regs <= 128 for regs, _, _ in ents.values()), ents
    # RES_STATIC_SMEM_D2 (resident.cuh, 10 KiB) is what the two-blocks-per-SM static_assert counts for these kernels
    smem = {}
    cur = None
    for line in log.read_text().splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", line)
        if m:
            cur = m.group(1)
        m = re.search(r"(\d+) bytes smem", line)
        if m and cur in D2.values():
            smem[cur] = int(m.group(1))
    assert set(smem) == set(D2.values()), smem
    assert all(v <= 10 * 1024 for v in smem.values()), smem


def _loops(sass):
    """(opcode counter) of every innermost backward-branch loop of a SASS listing"""
    ins = []
    for l in sass.splitlines():
        m = re.search(r"/\*([0-9a-f]{4,})\*/\s+(.*?);", l)
        if m:
            ins.append((int(m.group(1), 16), m.group(2).strip()))
    loops = []
    for a, t in ins:
        m = re.search(r"BRA\S*\s+.*?0x([0-9a-f]+)", t)
        if m and int(m.group(1), 16) < a:
            body = [x[1] for x in ins if int(m.group(1), 16) <= x[0] <= a]
            loops.append(collections.Counter(re.sub(r"^@!?U?P\w+\s+", "", x).split()[0] for x in body))
    return loops


@pytest.mark.parametrize("order", sorted(D2))
def test_staged_loop_stages_through_shared_memory(order):
    obj = _need(CSRC / "resident.o")
    cuobjdump = shutil.which("cuobjdump")
    if cuobjdump is None:
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", "-fun", D2[order], str(obj)], capture_output=True, text=True, timeout=600).stdout
    assert "UBLKCP" in sass
    # the tile loops: an mbarrier wait, bulk copies issued, the field products - and no reduction inside (REDUX only
    # after the loop). At least the eval-only, full-scalar bind and 125-bit bind variants.
    staged = [c for c in _loops(sass) if any(k.startswith("SYNCS.PHASECHK") for k in c) and any(k.startswith("UBLKCP") for k in c)
              and not any(k.startswith("REDUX") for k in c)]
    assert len(staged) >= 3, staged
    for c in staged:
        ops = set(c)
        assert not any(k.startswith(("LDL", "STL")) for k in ops), c       # no local memory
        assert not any(k.startswith(("LD.E", "ST.E")) for k in ops), c     # no generic loads / stores
        assert c["LDS.128"] >= 4                                           # operands come out of the staged tile
        assert sum(v for k, v in c.items() if k.startswith("IMAD.WIDE")) >= 60  # one 8 x 8-limb product per thread
