"""Random linear combinations on the device (jb_table_linear_combination, Polynomial.linear_combination) compared
bit-exactly with tests/lincomb_ref.py at small sizes and with the C restatement (tests/lincomb_cref.py) at scale; the
evaluation identity against the existing evaluation entry points, the commitment homomorphism against the existing
MSMs, a batched HyperKZG open of the combination, and every error of the contract, after which the context keeps
working."""
import ctypes

import numpy as np
import pytest

import jolt_b200
from jolt_b200 import (G1Bases, HyperKZG, LinearTerm, Polynomial, _lib, evaluate_small, g1_jacobian_to_affine,
                       one_hot_evaluate, small_scalars)
from jolt_b200 import field as F
from oracle import bn254 as O
import lincomb_cref as CR
import lincomb_ref as LR
import source_ref as SR
from gpu_util import EDGE_INTS, rand_limbs

pytestmark = pytest.mark.gpu
R = O.R_MOD
MAX125 = (1 << 125) - 1
G = np.array(O.to_mont_limbs(1, O.Q_MOD) + O.to_mont_limbs(2, O.Q_MOD), dtype=np.uint64)
LAYOUT = {"cycle_major": 0, "address_major": 1}
KINDS = ("u8", "u16", "u32", "u64", "u128", "i64", "i128", "s64", "s128")
NP_KIND = {"u8": np.uint8, "u16": np.uint16, "u32": np.uint32, "u64": np.uint64, "i64": np.int64}


@pytest.fixture(scope="module")
def sess():
    s = jolt_b200.Session(0)
    yield s
    s.close()


def coeff(i, seed):
    """0, 1, p - 1, a 125-bit challenge and random full-width values in turn."""
    return [0, 1, R - 1, MAX125 - seed % 1000, O.random_fr(seed, 1)[0]][i % 5]


def compact_values(kind, m, rng):
    """m entries of `kind` as small_scalars takes them, the extremes of the kind first."""
    if kind in NP_KIND:
        info = np.iinfo(NP_KIND[kind])
        v = rng.integers(info.min, info.max, m, dtype=NP_KIND[kind], endpoint=True)
        ext = [info.min, info.max, 0, 1] + ([-1] if kind == "i64" else [])
        v[: min(m, len(ext))] = ext[: min(m, len(ext))]
        return v
    if kind == "u128":
        v = [int(rng.integers(0, 1 << 63)) << int(rng.integers(0, 65)) for _ in range(m)]
        ext = [(1 << 128) - 1, 0, 1 << 127]
    elif kind == "i128":
        v = [int(rng.integers(-(1 << 62), 1 << 62)) << int(rng.integers(0, 65)) for _ in range(m)]
        ext = [-(1 << 127), (1 << 127) - 1, -1, 0]
    else:
        bits = 64 if kind == "s64" else 128
        v = [(int(rng.integers(0, 1 << 63)) << int(rng.integers(0, bits - 62)), bool(rng.integers(0, 2))) for _ in range(m)]
        ext = [(0, True), (0, False), ((1 << bits) - 1, False), ((1 << bits) - 1, True)]
    v[: min(m, len(ext))] = ext[: min(m, len(ext))]
    return v


def addresses(rng, T, K, dtype, none_frac):
    none = np.iinfo(dtype).max
    col = rng.integers(0, min(K, none), T).astype(dtype)
    col[rng.random(T) < none_frac] = none
    return col


class Terms:
    """One set of terms in the three forms: the device's LinearTerms, the big-int reference's (small sizes only) and
    the C oracle's. `big`: tables from numpy limbs, compact columns of numpy kinds and raw i128 device records."""

    def __init__(self, sess, seed, big=False):
        self.s, self.rng, self.seed, self.big = sess, np.random.default_rng(seed), seed, big
        self.dev, self.ref, self.cref, self.claims = [], [], [], []

    def _c(self):
        return coeff(len(self.dev), self.seed + len(self.dev))

    def table(self, n_i, values=None, poly=None):
        c = self._c()
        if poly is None:
            limbs = (F.ints_to_limbs(values if values is not None else O.random_fr(self.seed * 97 + len(self.dev), 1 << n_i))
                     if not self.big else rand_limbs(self.seed * 97 + len(self.dev), 1 << n_i))
            poly = Polynomial.new(self.s, limbs)
        else:
            limbs = next(t[1] for t in self.cref if t[0] == "table" and t[3] is poly)
        self.dev.append(LinearTerm.table(poly, c))
        if not self.big:
            self.ref.append(("table", F.limbs_to_ints(limbs), c))
        self.cref.append(("table", limbs, c, poly))
        self.claims.append(("table", poly, c))
        return poly

    def compact(self, kind, n_i, device=False):
        import torch
        c = self._c()
        if self.big and kind not in NP_KIND:   # raw two's-complement records, read in place on the device
            a = self.rng.integers(0, 1 << 64, size=(1 << n_i, 2), dtype=np.uint64)
            self.dev.append(LinearTerm.compact(torch.from_numpy(a.view(np.int64).copy()).cuda(), c, kind=kind))
            self.cref.append(("compact", a, _lib_kind(kind), 1 << n_i, c))
            return
        vals = compact_values(kind, 1 << n_i, self.rng)
        a, k, m = small_scalars(vals, kind if kind not in NP_KIND else None)
        if device:
            raw = a.view(np.int64) if kind not in ("u8", "i64") else a
            self.dev.append(LinearTerm.compact(torch.from_numpy(raw.copy()).cuda(), c, kind=kind))
        else:
            self.dev.append(LinearTerm.compact(vals, c, kind=kind if kind not in NP_KIND else None))
        if not self.big:
            self.ref.append(("compact", SR.decode_column(a, kind), c))
        self.cref.append(("compact", a, k, m, c))
        self.claims.append(("compact", (vals, kind), c))

    def one_hot(self, dtype, K, lt, layout, none_frac=0.3, device=False):
        c = self._c()
        col = addresses(self.rng, 1 << lt, K, dtype, none_frac)
        if device:
            import torch
            src = torch.from_numpy(col.copy() if dtype == np.uint8 else col.view(np.int16).copy()).cuda()
            self.dev.append(LinearTerm.one_hot(src, K, c, layout))
        else:
            self.dev.append(LinearTerm.one_hot(col, K, c, layout))
        if not self.big:
            self.ref.append(("one_hot", SR.addresses(col), K, layout, c))
        self.cref.append(("one_hot", col, K, LAYOUT[layout], c))
        self.claims.append(("one_hot", (col, K, layout), c))

    def cterms(self):
        return [t[:3] if t[0] == "table" else t for t in self.cref]

    def check_inputs(self):
        for t in self.cref:
            if t[0] == "table":
                assert np.array_equal(t[3].evals(), t[1])


def _lib_kind(kind):
    from jolt_b200 import SCALAR_KINDS
    return SCALAR_KINDS[kind]


def mixed(sess, n, seed, device=False):
    """Every compact kind, one-hot u8 / u16 in both layouts, shorter terms, a repeated handle and edge values."""
    t = Terms(sess, seed)
    rng = np.random.default_rng(seed)
    edge = t.table(n, values=[EDGE_INTS[i] for i in rng.integers(0, len(EDGE_INTS), 1 << n)])
    t.table(max(n - 1, 0))
    t.table(n, poly=edge)                 # the same handle again
    for i, kind in enumerate(KINDS):
        t.compact(kind, n if i % 2 == 0 else max(n - 2, 0), device)
    if n >= 1:
        t.one_hot(np.uint8, 2, n - 1, "cycle_major", device=device)
        t.one_hot(np.uint16, 1 << (n // 2), n - n // 2, "address_major", device=device)
        t.one_hot(np.uint8, 1, max(n - 2, 0), "address_major", none_frac=1.0, device=device)
    return t


@pytest.mark.parametrize("n", [0, 1, 2, 5, 10, 14])
def test_matches_reference(sess, n):
    t = mixed(sess, n, 100 + n)
    P = Polynomial.linear_combination(sess, t.dev)
    assert len(P) == 1 << n
    assert P.to_ints() == LR.linear_combination(t.ref, 1 << n)
    t.check_inputs()
    longer = Polynomial.linear_combination(sess, t.dev, length=1 << (n + 1))
    assert longer.to_ints() == LR.linear_combination(t.ref, 1 << (n + 1))


@pytest.mark.parametrize("layout", ["cycle_major", "address_major"])
@pytest.mark.parametrize("dtype,K,lt", [(np.uint8, 1, 6), (np.uint8, 2, 6), (np.uint8, 16, 5), (np.uint8, 256, 3),
                                        (np.uint16, 1, 6), (np.uint16, 16, 5), (np.uint16, 256, 3),
                                        (np.uint16, 1 << 16, 2)])
@pytest.mark.parametrize("none_frac", [0.0, 0.3, 1.0])
def test_one_hot(sess, dtype, K, lt, layout, none_frac):
    t = Terms(sess, K + lt)
    t.one_hot(dtype, K, lt, layout, none_frac)
    t.one_hot(dtype, K, lt, layout, none_frac)
    t.dev[0] = LinearTerm.one_hot(t.cref[0][1], K, MAX125, layout)
    t.ref[0] = t.ref[0][:-1] + (MAX125,)
    t.cref[0] = t.cref[0][:-1] + (MAX125,)
    got = Polynomial.linear_combination(sess, t.dev).to_ints()
    want = (LR.linear_combination(t.ref, K << lt) if K <= 256 else
            F.limbs_to_ints(CR.linear_combination(t.cterms(), K << lt)))
    assert got == want


def test_host_and_device_columns_agree(sess):
    n = 12
    host, dev = mixed(sess, n, 7), mixed(sess, n, 7, device=True)
    a = Polynomial.linear_combination(sess, host.dev).evals()
    b = Polynomial.linear_combination(sess, dev.dev).evals()
    assert np.array_equal(a, b)


@pytest.mark.parametrize("kind", ["u128", "s128"])
def test_device_records_need_only_8_byte_alignment(sess, kind):
    """A device column is aligned to min(8, entry bytes): 16- and 24-byte records at base + 8 are read in place."""
    import torch
    n, c = 6, coeff(4, 9)
    vals = compact_values(kind, 1 << n, np.random.default_rng(9))
    a, _, _ = small_scalars(vals, kind)
    buf = torch.zeros(a.size + 8, dtype=torch.int64, device="cuda")
    off = next(o for o in range(1, 8) if (buf.data_ptr() + 8 * o) % 16 and (buf.data_ptr() + 8 * o) % 24)
    col = buf[off:off + a.size]
    col.copy_(torch.from_numpy(a.view(np.int64).reshape(-1).copy()))
    P = Polynomial.linear_combination(sess, [LinearTerm.compact(col, c, kind=kind)])
    assert P.to_ints() == LR.linear_combination([("compact", SR.decode_column(a, kind), c)], 1 << n)
    pt = O.random_fr(10, n)
    assert evaluate_small(sess, col, pt, kinds=kind) == evaluate_small(sess, [vals], pt, kinds=kind)


def _scale_terms(sess, n, count, seed, one_hot_K=16):
    t = Terms(sess, seed, big=True)
    kinds = ["u8", "u64", "i128", "i64", "u16", "s64"]
    for i in range(count):
        r = i % 4
        if r == 0:
            t.table(n - (i % 3))
        elif r == 1:
            t.compact(kinds[i % len(kinds)], n - (i % 2))
        elif r == 2 and one_hot_K:
            t.one_hot(np.uint8 if i % 8 == 2 else np.uint16, one_hot_K, n - one_hot_K.bit_length() + 1,
                      "cycle_major" if i % 8 == 2 else "address_major")
        else:
            t.table(n, poly=t.claims[0][1])
    return t


@pytest.mark.parametrize("n,count", [(22, 16), (24, 8), (16, 200)])
def test_at_scale_against_c_oracle(sess, n, count):
    t = _scale_terms(sess, n, count, 300 + n)
    P = Polynomial.linear_combination(sess, t.dev)
    assert np.array_equal(P.evals(), CR.linear_combination(t.cterms(), 1 << n))
    t.check_inputs()


def test_evaluation_identity(sess):
    """P(point) = sum_i c_i prod(1 - point_hi) e_i, each e_i from the independent evaluation entry points"""
    n = 14
    t = mixed(sess, n, 55)
    point = O.random_fr(56, n)
    P = Polynomial.linear_combination(sess, t.dev)
    claims = []
    for kind, what, c in t.claims:
        if kind == "table":
            n_i = what.num_vars()
            e = what.evaluate(point[n - n_i:])
        elif kind == "compact":
            vals, k = what
            n_i = len(vals).bit_length() - 1
            e = evaluate_small(sess, vals if k in ("u8", "u16", "u32", "u64", "i64") else [vals],
                               point[n - n_i:], kinds=None if k in NP_KIND else k)[0]
        else:
            col, K, layout = what
            n_i = (K * col.shape[0]).bit_length() - 1
            e = one_hot_evaluate(sess, col, K, point[n - n_i:], layout)[0]
        claims.append((c, n_i, e))
    assert P.evaluate(point) == LR.combined_claim(claims, point)


def _commitments(bases, t):
    """C_i of every term from the existing MSM entry points (affine)."""
    out = []
    for kind, what, c in t.claims:
        if kind == "table":
            C = bases.msm(what)
        elif kind == "compact":
            vals, k = what
            C = bases.msm_small(vals, kind=None if k in NP_KIND else k)
        else:
            col, K, layout = what
            C = bases.one_hot_rows(col, K, K * col.shape[0], layout)[0, 0]
        out.append((c, g1_jacobian_to_affine(C)))
    return out


def test_commitment_homomorphism_2_12(sess):
    n = 12
    bases = G1Bases.generate_multiples(sess, G, 1 << n)
    t = mixed(sess, n, 77)
    P = Polynomial.linear_combination(sess, t.dev)
    acc = None
    for c, Ci in _commitments(bases, t):
        acc = O.g1_add(acc, O.g1_scalar_mul(Ci, c) if Ci is not None else None)
    assert g1_jacobian_to_affine(bases.msm(P)) == acc


def test_commitment_homomorphism_2_20_closed_form(sess):
    """bases (i + 1) G: commit(p) = (sum_x (x + 1) p[x]) G, so the homomorphism is an identity on those scalars"""
    n = 20
    bases = G1Bases.generate_multiples(sess, G, 1 << n)
    t = _scale_terms(sess, n, 8, 20)
    P = Polynomial.linear_combination(sess, t.dev)

    def weight(vals):
        return sum((x + 1) * v for x, v in enumerate(vals)) % R

    s = weight(P.to_ints())
    want = 0
    for term in t.cterms():
        alone = term[:-1] + (1,)
        n_i = (term[1].shape[0] * (term[2] if term[0] == "one_hot" else 1)).bit_length() - 1
        want += (term[-1] % R) * weight(F.limbs_to_ints(CR.linear_combination([alone], 1 << n_i)))
    assert s == want % R
    gen = (O.from_mont_limbs(G[:4], O.Q_MOD), O.from_mont_limbs(G[4:], O.Q_MOD))
    assert g1_jacobian_to_affine(bases.msm(P)) == O.g1_scalar_mul(gen, s)


@pytest.mark.parametrize("ell", [10, 20])
def test_batched_open(sess, ell):
    bases = G1Bases.generate_multiples(sess, G, 1 << ell)
    t = _scale_terms(sess, ell, 10, 40 + ell)
    P_dev = Polynomial.linear_combination(sess, t.dev)
    P_host = Polynomial.new(sess, CR.linear_combination(t.cterms(), 1 << ell))
    point = F.ints_to_limbs(O.random_fr(41, ell))
    r_int, q_int = O.random_fr(42, 2)
    a = HyperKZG.open(bases, P_dev, point, lambda com: r_int, lambda v: q_int)
    b = HyperKZG.open(bases, P_host, point, lambda com: r_int, lambda v: q_int)
    assert [g1_jacobian_to_affine(x) for x in a.com] == [g1_jacobian_to_affine(x) for x in b.com]
    assert [g1_jacobian_to_affine(x) for x in a.w] == [g1_jacobian_to_affine(x) for x in b.w]
    assert a.v == b.v


# ---- errors ----------------------------------------------------------------------------------------------------------
def _raw(sess, terms, count=None, length=4):
    arr = (_lib.LcTermC * max(len(terms), 1))()
    for i, t in enumerate(terms):
        arr[i] = t
    out = ctypes.c_uint64(0)
    st = sess.lib.jb_table_linear_combination(sess.h, ctypes.cast(arr, ctypes.c_void_p),
                                              len(terms) if count is None else count, length, ctypes.byref(out))
    return st, out.value


def _term(**kw):
    t = _lib.LcTermC()
    t.type = kw.get("type", _lib.JB_LC_COMPACT)
    t.kind = kw.get("kind", 1)
    t.on_device = kw.get("on_device", 0)
    t.layout = kw.get("layout", 0)
    t.table = kw.get("table", 0)
    t.values = kw.get("values", None)
    t.len = kw.get("len", 4)
    t.K = kw.get("K", 1)
    t.coeff[:] = [int(x) for x in kw.get("coeff", F.to_limbs(3))]
    return t


def test_errors_leave_the_context_usable(sess):
    u8 = np.array([1, 2, 3, 4], dtype=np.uint8)
    u16 = np.array([0, 1, 0xFFFF, 3], dtype=np.uint16)
    poly = Polynomial.from_ints(sess, [5, 6, 7, 8])
    odd_h = ctypes.c_uint64()
    sess.check(sess.lib.jb_table_alloc(sess.h, 3, ctypes.byref(odd_h)))
    odd = Polynomial(sess, odd_h.value)
    before = poly.evals().copy()
    vp = u8.ctypes.data
    INV, UNS = _lib.JB_ERR_INVALID, _lib.JB_ERR_UNSUPPORTED
    import torch
    dev16 = torch.zeros(8, dtype=torch.int16, device="cuda")
    cases = [
        ([], 0, 4, INV),                                                                  # count == 0
        ([_term(type=7, values=vp)], None, 4, INV),                                      # unknown type
        ([_term(kind=0, values=vp)], None, 4, INV),                                      # FR is not compact
        ([_term(kind=10, values=vp)], None, 4, INV),                                     # unknown kind
        ([_term(values=vp)], None, 3, INV),                                              # len not a power of two
        ([_term(values=vp)], None, 2, INV),                                              # term longer than len
        ([_term(values=vp, len=3)], None, 4, INV),                                       # term length
        ([_term(values=None)], None, 4, INV),                                            # null column
        ([_term(values=vp, on_device=2)], None, 4, INV),                                 # on_device
        ([_term(values=vp, coeff=[int(x) for x in F.to_limbs(0)][:3] + [0xFFFFFFFFFFFFFFFF])], None, 4, INV),
        ([_term(type=_lib.JB_LC_TABLE, table=123456789)], None, 4, INV),                 # unknown handle
        ([_term(type=_lib.JB_LC_TABLE, table=odd.handle)], None, 4, INV),                # table length
        ([_term(kind=4, values=dev16.data_ptr() + 2, on_device=1)], None, 4, INV),       # misaligned device column
        ([_term(type=_lib.JB_LC_ONE_HOT, kind=4, values=vp)], None, 4, INV),             # one-hot kind
        ([_term(type=_lib.JB_LC_ONE_HOT, layout=2, values=vp)], None, 4, INV),           # layout
        ([_term(type=_lib.JB_LC_ONE_HOT, K=3, values=vp)], None, 16, INV),               # K
        ([_term(type=_lib.JB_LC_ONE_HOT, K=4, values=vp)], None, 8, INV),                # K T > len
        ([_term(type=_lib.JB_LC_ONE_HOT, kind=2, K=2, values=dev16.data_ptr() + 1, on_device=1)], None, 8, INV),
        ([_term(type=_lib.JB_LC_ONE_HOT, kind=2, K=1 << 17, values=u16.ctypes.data)], None, 1 << 20, UNS),
        ([_term(type=_lib.JB_LC_ONE_HOT, kind=2, K=1, len=1 << 31, values=u16.ctypes.data)], None, 1 << 31, UNS),
        ([_term(type=_lib.JB_LC_ONE_HOT, K=2, values=vp)], None, 8, INV),                # address 2..4 >= K = 2
        ([_term(type=_lib.JB_LC_ONE_HOT, kind=2, K=2, values=u16.ctypes.data)], None, 8, INV),  # address 3 >= 2
    ]
    good = [_term(type=_lib.JB_LC_TABLE, table=poly.handle, coeff=F.to_limbs(2)), _term(values=vp)]
    for i, (terms, count, length, want) in enumerate(cases):
        st, h = _raw(sess, terms, count, length)
        assert st == want, (i, st, sess.lib.jb_last_error(sess.h))
        assert h == 0, i
        st, h = _raw(sess, good)
        assert st == _lib.JB_OK, i
        assert Polynomial(sess, h).to_ints() == [(2 * a + 3 * b) % R for a, b in zip([5, 6, 7, 8], [1, 2, 3, 4])]
        Polynomial(sess, h).free()
    assert sess.lib.jb_table_linear_combination(sess.h, None, 1, 4, ctypes.byref(ctypes.c_uint64())) == INV
    assert np.array_equal(poly.evals(), before)
    with pytest.raises(ValueError):
        Polynomial.linear_combination(sess, [])
