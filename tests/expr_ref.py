"""Python big-int reference for expression members: the round polynomials of
    sum_x [eq(w, x) *] sum_k c_k prod_i f_{tables_k[i]}(x)
for monomials [(c_k, [table indices])] over multilinear tables, and an oracle member with the ProductMember interface
of oracle/bn254.py (so it drives O.prove_batch). Pinned against brute force over the hypercube by
tests/test_expr_ref_cpu.py."""
import math

from oracle import bn254 as O

P = O.R_MOD


def expr_value(vals: list[int], monomials) -> int:
    """sum_k c_k prod_i vals[tables_k[i]] mod p"""
    return sum(c * math.prod(vals[t] for t in tabs) for c, tabs in monomials) % P


def expr_degree(monomials, eq: bool) -> int:
    return max(len(tabs) for _, tabs in monomials) + (1 if eq else 0)


def _round_evals(tables, monomials, order, eq_table):
    """s(t), t = 0..degree, of the current round from the current (partly bound) tables and eq table."""
    deg = expr_degree(monomials, eq_table is not None)
    half = len(tables[0]) // 2
    out = [0] * (deg + 1)
    for y in range(half):
        pairs = [O.pair(t, y, order) for t in tables]
        e = O.pair(eq_table, y, order) if eq_table is not None else None
        for t in range(deg + 1):
            v = expr_value([lo + t * (hi - lo) for lo, hi in pairs], monomials)
            if e is not None:
                v = v * (e[0] + t * (e[1] - e[0]))
            out[t] += v
    return [v % P for v in out]


def expr_round_evals(tables, monomials, order, eq_point=None, eq_scale=None):
    """Evaluations at t = 0..degree of the first round polynomial of the expression member over `tables` (lists of
    ints); with `eq_point` the summand carries eq(eq_point, x) * eq_scale (eq_point[0] <-> the index MSB)."""
    eq_table = None if eq_point is None else O.eq_evals(list(eq_point), eq_scale)
    return _round_evals([list(t) for t in tables], monomials, order, eq_table)


class ExpressionMember:
    """Reference-tier expression member (interface of oracle.bn254.ProductMember): binds every table (and the
    materialised eq table) per challenge and sums the expression over the pairs. prove_round checks s(0) + s(1)
    against the claim and returns the coefficients."""

    def __init__(self, tables, monomials, order=O.HIGH_TO_LOW, eq_point=None, eq_scale=None):
        self.tables = [[v % P for v in t] for t in tables]
        self.monomials = [(c % P, list(tabs)) for c, tabs in monomials]
        self.order = order
        self.eq = None if eq_point is None else O.eq_evals(list(eq_point), eq_scale)
        self.rounds = len(self.tables[0]).bit_length() - 1
        self.degree = expr_degree(self.monomials, self.eq is not None)

    def num_rounds(self):
        return self.rounds

    def _bind(self, c):
        self.tables = [O.bind(t, c, self.order) for t in self.tables]
        if self.eq is not None:
            self.eq = O.bind(self.eq, c, self.order)

    def round_evals(self, bind_c):
        if bind_c is not None:
            self._bind(bind_c)
        return _round_evals(self.tables, self.monomials, self.order, self.eq)

    def prove_round(self, bind_c, rnd, previous_claim):
        ev = self.round_evals(bind_c)
        if (ev[0] + ev[1]) % P != previous_claim % P:
            raise ValueError(f"RoundCheckFailed round={rnd}")
        return O.uni_from_evals(ev)

    def finish_rounds(self, bind_c):
        self._bind(bind_c)

    def final_evals(self):
        return [t[0] for t in self.tables]

    def eq_scalar(self):
        return self.eq[0]

    def claim(self):
        """sum_x of the summand over the current tables"""
        ev = _round_evals(self.tables, self.monomials, self.order, self.eq)
        return (ev[0] + ev[1]) % P
