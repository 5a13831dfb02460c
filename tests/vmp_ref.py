"""Big-int reference for Dory's vector-matrix product (jb_lc_vector_matrix_product): the joint polynomial P of
tests/lincomb_ref.py laid out as R = length / W rows of W columns (flat index x = row W + col), combined by rows:
    v[col] = sum_{row < R} left[row] P[row W + col]
Pinned by tests/test_vmp_cpu.py against a brute-force double sum and the materialised one-hot matrix;
tests/test_gpu_vmp.py compares the device against it."""
import lincomb_ref as LR

P = LR.P


def vector_matrix_product(terms, length: int, W: int, left) -> list[int]:
    assert length % W == 0 and len(left) == length // W
    joint = LR.linear_combination(terms, length)
    return [sum(left[r] * joint[r * W + c] for r in range(len(left))) % P for c in range(W)]
