"""CPU oracle for the large-steps hot path  --  TEST INFRASTRUCTURE ONLY.

This package is a numpy/scipy restatement of the reference's algorithm for the path
    compute_matrix -> to_differential -> from_differential (solve M x = b, fwd + bwd) -> AdamUniform.step
Each function cites the reference file:line it follows (paths relative to the reference repository root).

Only `tests/`, `__graft_entry__.smoke()` and the `cpu_baseline` / `--impl reference` legs of
`bench.py` may import it, and only as the checker / CPU baseline -- never on the product path.
The product (`large-steps-pytorch_b200/largesteps_b200`) fails loudly when its CUDA library is missing.

Parity pinning status
  * assembly (`geometry.py:3-133`), reference CG (`solvers.py:41-126`), AdamUniform (`optimize.py:17-41`),
    to_differential (`parameterize.py:30`): PINNED against outputs of the unmodified reference run on the
    CPU (tests/golden/make_golden.py -> tests/golden/*.npz; checked by tests/test_oracle.py).
  * oracle/cg_port.c (+ cport.py): the reference CG once more in plain C with OpenMP, pinned against the same golden
    outputs (tests/test_oracle.py); it is the multi-threaded CPU baseline of bench.py.
  * Cholesky path (`solvers.py:26-39`): the arithmetic lives in the third-party wheel `cholespy`
    (requirements.txt:1 `cholespy>=0.1.4`, not vendored, not installable offline) -- PARITY UNPINNED at that
    boundary.  It is a direct solve of M x = b, so the oracle is an fp64 sparse direct solve (SuperLU,
    symmetric mode; dense Cholesky for small V) and the bar is rel-L2 <= 1e-5 against it.
"""
from .assembly import laplacian_uniform, laplacian_cot, compute_matrix, coo_to_scipy  # noqa: F401
from .solve import (DirectSolver, dense_cholesky_solve, reference_cg, ReferenceCG,     # noqa: F401
                    to_differential, jacobi_pcg_f32, fused_pcg_f32, gershgorin_bound, chebyshev_coefficients)
from .adam import AdamUniformOracle  # noqa: F401
# oracle.cport.CPortCG: OpenMP C restatement of the reference CG (oracle/cg_port.c), built on demand with gcc
# sell_spmv_f32: exact model of the solver's SELL-32 SpMV (same file); sell32: each row's padded width in that copy
from .cport import sell32, sell_spmv_f32  # noqa: F401
