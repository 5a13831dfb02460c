"""u32 address columns without a GPU: the Python entry points that take them opt in and the others still refuse them,
the limits live in one place (columns.cuh), only the entry points that accept u32 load it, the references of
tests/u32_ref.py agree with the flat ones of tests/mle_eval_ref.py and keep the read-write precondition, and the static budgets of the kernels that now read u32 columns."""
import pathlib
import re

import numpy as np
import pytest

from jolt_b200 import api
from oracle import bn254 as O
import mle_eval_ref as M
import u32_ref as U
from test_build_artifacts import ptxas_entries

CSRC = pathlib.Path(__file__).resolve().parents[1] / "jolt_b200" / "csrc"


def test_address_columns_take_u32_only_on_request():
    col = np.array([0, 5, 0xFFFFFFFF, (1 << 24) - 1], dtype=np.uint32)
    with pytest.raises(ValueError, match="one_hot_rows"):
        api._address_columns(col, "one_hot_rows")
    ptrs, kind, T, dev, _keep = api._address_columns([col, col.copy()], "one_hot_evaluate", u32=True)
    assert kind == api.SCALAR_KINDS["u32"] and T == 4 and dev == 0 and len(ptrs) == 2
    for dt, k in ((np.uint8, "u8"), (np.uint16, "u16")):
        assert api._address_columns(col.astype(dt), "x", u32=True)[1] == api.SCALAR_KINDS[k]
    with pytest.raises(ValueError):   # one dtype for all columns
        api._address_columns([col, col.astype(np.uint16)], "x", u32=True)
    with pytest.raises(ValueError):   # signed host arrays are not address columns
        api._address_columns(col.view(np.int32), "x", u32=True)
    assert api.ONE_HOT_NONE[np.dtype(np.uint32)] == 0xFFFFFFFF


def test_one_limit_in_columns_cuh():
    src = (CSRC / "columns.cuh").read_text()
    assert "constexpr size_t ONE_HOT_MAX_K_U32 = (size_t)1 << 24;" in src
    assert "constexpr size_t ONE_HOT_MAX_K = (size_t)1 << 16;" in src
    # the entry points that take u32 ask for it; booleanity, linear combinations, VMP and one_hot_rows do not
    wide = {"mle_eval.cu": 2, "read_write.cu": 1}
    for f in sorted(CSRC.glob("*.cu*")):
        text = f.read_text()
        n = len(re.findall(r"check_one_hot_columns\([^;]*SK_U32\)", text))
        assert n == wide.get(f.name, 0), (f.name, n)
        if f.name in ("booleanity.cu", "lincomb.cu", "vmp.cu", "msm.cu", "lc_terms.cuh"):
            assert "ld_address<SK_U32>" not in text, f.name
    assert "ADDRESS_WIDEST = SK_U16" in (CSRC / "sources.cu").read_text()
    assert "ADDRESS_WIDEST = SK_U32" in (CSRC / "product.cu").read_text()


@pytest.mark.parametrize("K,T", [(1, 4), (4, 8), (16, 16), (64, 8)])
def test_sparse_references_equal_the_flat_ones(K, T):
    rng = np.random.default_rng(K + T)
    addr = [None if rng.random() < 0.25 else int(a) for a in rng.integers(0, K, T)]
    lt, lk = T.bit_length() - 1, K.bit_length() - 1
    r_cycle, r_addr = O.random_fr(K * T, lt), O.random_fr(K * T + 1, lk)
    assert U.one_hot_evaluate_sparse(addr, r_cycle, r_addr) == M.one_hot_evaluate(addr, K, T, r_cycle + r_addr,
                                                                                     "cycle_major")
    G = M.pushforward(addr, K, r_cycle)
    sparse = U.pushforward_sparse(addr, r_cycle)
    assert all(G[k] == sparse.get(k, 0) for k in range(K))
    eq = O.eq_evals(r_addr) if lk else [1]
    assert [U.eq_at(r_addr, k) for k in range(K)] == eq


def test_u32_columns_workload_keeps_the_precondition():
    K, T = 1 << 20, 1 << 12
    for local in (False, True):
        wl = U.ram_columns_workload_u32(5, K, T, local=local)
        a = wl["addrs"][0]
        assert a.dtype == np.uint32 and wl["none"] == 0xFFFFFFFF
        hit = a != 0xFFFFFFFF
        assert (a[hit] < K).all()
        # Val(k, j) by a running table over the touched addresses
        cur = {}
        for j in range(T):
            k = int(a[j])
            if k == 0xFFFFFFFF:
                assert wl["values"][0][j] == 0 and wl["inc"][j] == 0
                continue
            v = cur.get(k, int(wl["init"][k]))
            assert int(wl["values"][0][j]) == v
            cur[k] = v + int(wl["inc"][j])
        if local:   # a walk: most touched addresses are near the previous one
            steps = np.diff(a[hit].astype(np.int64)) % K
            assert np.mean(np.minimum(steps, K - steps) <= 4) > 0.9


def test_rw_workload_edges():
    K, T, accesses, *_ = U.ram_workload_with_edges(3, 1 << 17, 16)
    assert accesses[0][0][0] == 0 and accesses[0][0][1] == K - 1


def _need(p):
    if not p.exists():
        pytest.skip("no build in this tree yet (python -c 'import __graft_entry__ as g; g.build()')")
    return p


def test_kernels_that_read_u32_stay_within_budget():
    ents = {k: v for k, v in ptxas_entries(_need(CSRC / "mle_eval.ptxas.log")).items() if "pushforward_kernel" in k}
    assert len(ents) == 4 and all(r <= 128 and (s, l) == (0, 0) for r, s, l in ents.values()), ents
    src = {k: v for k, v in ptxas_entries(_need(CSRC / "sources.ptxas.log")).items() if "check_addresses_kernel" in k}
    assert len(src) == 2 and all((s, l) == (0, 0) for _, s, l in src.values()), src
    prod = {k: v for k, v in ptxas_entries(_need(CSRC / "product.ptxas.log")).items()
            if "product_round_kernel" in k or "source_bind_kernel" in k}
    assert len(prod) == 22 and all((s, l) == (0, 0) for _, s, l in prod.values()), prod
    rw = {k: v for k, v in ptxas_entries(_need(CSRC / "read_write.ptxas.log")).items()
          if "rw_count_kernel" in k or "rw_fill_kernel" in k}
    assert len(rw) == 8 and all((s, l) == (0, 0) for _, s, l in rw.values()), rw
