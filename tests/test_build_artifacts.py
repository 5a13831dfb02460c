"""Static checks on the built device code (no GPU): the hot kernels keep their resource budget and their 128-bit
memory instructions (the widest sm_90 has). Reads the ptxas logs / objects `make -C jolt_b200/csrc` leaves in-tree; skipped before a build."""
import pathlib
import re
import shutil
import subprocess

import pytest

CSRC = pathlib.Path(__file__).resolve().parents[1] / "jolt_b200" / "csrc"


def ptxas_entries(log: pathlib.Path) -> dict:
    """mangled kernel name -> (registers, spill_store_bytes, spill_load_bytes)"""
    out, cur, spills = {}, None, (0, 0)
    for line in log.read_text().splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", line)
        if m:
            cur = m.group(1)
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur:
            spills = (int(m.group(1)), int(m.group(2)))
        m = re.search(r"Used (\d+) registers", line)
        if m and cur:
            out[cur] = (int(m.group(1)),) + spills
            cur = None
    return out


def _log(name):
    log = CSRC / name
    if not log.exists():
        pytest.skip("no build in this tree yet (python -c 'import __graft_entry__ as g; g.build()')")
    return ptxas_entries(log)


@pytest.fixture(scope="module")
def member_log():
    return _log("member.ptxas.log")


def test_every_fused_round_kernel_fits_two_blocks_per_sm_without_spills(member_log):
    # every instance is launched at 256 threads x 2 blocks/SM -> at most 128 registers, no local memory
    main = {k: v for k, v in member_log.items() if "fused_round_kernel" in k}
    assert len(main) >= 16
    for name, (regs, st, ld) in main.items():
        assert regs <= 128, (name, regs)
        # products of <= 2 tables (the bench configuration and the reference's common relations) must not touch local
        # memory at all; M = 3, 4 and the two-term sum of products carry a few spilled words at 128 registers - bounded
        if re.search(r"fused_round_kernelILi[12]ELi1ELi[01]E", name):
            assert (st, ld) == (0, 0), (name, st, ld)
        else:
            assert st <= 128 and ld <= 128, (name, st, ld)


def test_resident_kernels_fit_two_blocks_per_sm():
    # the resident kernel is launched cooperatively at 2 blocks/SM: it must stay within 128 registers; the round loop
    # around the (out-of-line) passes may spill a few dozen words (touched once per ROUND, not per pair)
    ents = {k: v for k, v in _log("resident.ptxas.log").items() if "resident_rounds_kernel" in k}
    assert len(ents) >= 10
    for name, (regs, st, ld) in ents.items():
        assert regs <= 128, (name, regs)
        assert st <= 160 and ld <= 320, (name, st, ld)


def test_fused_round_kernel_uses_128_bit_memory_instructions():
    obj = CSRC / "member.o"
    cuobjdump = shutil.which("cuobjdump")
    if not obj.exists() or cuobjdump is None:
        pytest.skip("member.o or cuobjdump not available")
    fn = "_ZN2jb18fused_round_kernelILi2ELi1ELi1ELb1ELb1ELb1ELb0EEEvNS_9TablePtrsEmNS_10BindScalarENS_8RoundOutE"
    sass = subprocess.run([cuobjdump, "-sass", "-fun", fn, str(obj)], capture_output=True, text=True, timeout=300).stdout
    # an element (32 B) is two 128-bit requests: every read-only table load and the bound-value stores are 128 bits wide
    assert sass.count("LDG.E") >= 16 and all(".128" in l for l in sass.splitlines() if "LDG.E" in l and "CONSTANT" in l)
    assert any("STG.E" in l and ".128" in l for l in sass.splitlines())
    assert "IMAD.WIDE.U32" in sass                      # the 32x32+64 multiplier is the unit of work
    assert "LDL" not in sass and "STL" not in sass      # no local-memory traffic in the hot kernel
