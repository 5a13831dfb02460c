"""jolt_b200 - H100 (sm_90a) backend for the a16z/jolt prover hot path.

Python surface = thin ctypes bindings over the C ABI (include/jolt_b200.h) that mirror the
reference's Rust types for this path:
  Polynomial / DensePolynomial  crates/jolt-poly/src/dense.rs:35, jolt-prover-legacy/src/poly/dense_mlpoly.rs:20
  EqPolynomial                  crates/jolt-poly/src/eq.rs:24
  UnivariatePoly                crates/jolt-poly/src/univariate.rs:27
  ProveRounds / prove_batch     crates/jolt-sumcheck/src/prover.rs:52, :193
  msm / HyperKZG                crates/jolt-crypto/src/ec/group.rs:70, crates/jolt-hyperkzg/src/scheme.rs:275-338
The compute is CUDA only; importing this package requires the built extension."""
from ._lib import JoltB200Error, load  # noqa: F401
from .api import (  # noqa: F401
    HIGH_TO_LOW,
    LOW_TO_HIGH,
    ONE_HOT_LAYOUTS,
    ONE_HOT_NONE,
    SCALAR_KINDS,
    Source,
    BatchMember,
    EqPlusOnePolynomial,
    EqPolynomial,
    EqProductMember,
    ExpressionMember,
    G1Bases,
    HyperKZG,
    HyperKZGProof,
    LinearTerm,
    LtPolynomial,
    Polynomial,
    ProductMember,
    ProductSourcesMember,
    ProvedBatch,
    ReadWriteCheckingMember,
    BooleanityMember,
    RoundScheduler,
    Session,
    SumOfProductsMember,
    SumcheckError,
    UnivariatePoly,
    evaluate_small,
    g1_affine_limbs,
    g1_jacobian_to_affine,
    msm,
    one_hot_evaluate,
    one_hot_pushforward,
    point_limbs,
    prove_batch,
    prove_batch_native,
    small_scalars,
)

DensePolynomial = Polynomial  # legacy name (jolt-prover-legacy/src/poly/dense_mlpoly.rs:20)
load()
