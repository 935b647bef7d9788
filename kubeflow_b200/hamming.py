"""skopt's HammingKernel for all-categorical spaces, served by the engine's RBF kernel on the one-hot columns.

skopt's GP on a space whose every dimension is ``Categorical`` uses ``ConstantKernel * HammingKernel`` [RECALL]:
``k(x, y) = exp(−Σ_j l_j·[x_j ≠ y_j])`` over the category values, with per-dimension weights ``l_j`` (they multiply the
mismatch; skopt calls them length scales) bounded by (1e-5, 1e5).  ``Space`` one-hot encodes a dimension of c ≥ 3 categories
into c columns and a two-category dimension into one 0/1 column, and the engine's RBF kernel is ``exp(−½ Σ_c (Δ_c/ℓ_c)²)``.
A mismatch in dimension j gives Σ_c Δ_c² = 2 over its columns when c ≥ 3 and 1 when c = 2, so the RBF kernel with the
column length scales

    ℓ_c = l_j^(−1/2)        (c ≥ 3)          ℓ_c = (2·l_j)^(−1/2)        (c = 2)

is the Hamming kernel exactly, provided every row is encoded alike.  A one-category dimension has one column, which
``Categorical.to_unit`` (told rows, lies, the request scan) sets to 1 while ``Space.rvs_transformed`` writes the category index
0 into it; ``candidates`` therefore sets that column of the sampled candidates to 1, so it never differs, and its ℓ_c is held
at 1 whatever l_j is: the column contributes nothing to any kernel value or to the norms the tensor-core K* works from, and
that l_j has a zero gradient (skopt leaves it at its start).  Since log ℓ_c = −½ log l_j + const,
∂/∂log l_j = −½ Σ_{c ∈ j} ∂/∂log ℓ_c.

``HammingMap.length_scale`` is the one place that mapping is made: the Optimizer's fixed θ, its fit and the batched
θ evaluations all go through it, so every engine call (fit, append, rebase, sweep, LML gradient) serves the Hamming kernel;
``HammingMap.candidates`` is the one place the candidates' encoding is aligned with the told rows'.

The sweep.  The tensor-core suggestion path has been tested over kernel arguments (the RBF exponent ½ Σ_c (Δ_c/ℓ_c)² between
the two most distant points of the space) from about 0.22 to 139: length scales 0.2× to 5× the default on [0, 1]^8.  The
Hamming weights reach far outside that — l_j = 1e5 puts Δ_c/ℓ_c at about 450 — where the fp32 distances of the tensor-core
K* lose all accuracy near an exact match, and l_j → 1e-5 makes every kernel value nearly equal.  ``var_mode`` "auto"
therefore keeps the tensor-core path only while the largest kernel argument S = Σ_{j: c_j ≥ 2} l_j lies in ``TC_RANGE``, and
routes any other θ to the FP64 path (``var_mode`` "f64"); an explicit "tc" or "f64" is passed through.
"""
from __future__ import annotations

import numpy as np

from .space import Categorical

LS_BOUNDS = (1e-5, 1e5)          # HammingKernel's default length_scale_bounds [RECALL]
# S = Σ l_j over the dimensions with two or more categories, where "auto" may use the tensor cores.  The upper end is measured
# (DESIGN §7): the tensor-core pick held at S = 64 and missed the FP64 maximiser at S = 125.
TC_RANGE = (0.25, 32.0)


class HammingMap:
    """The column length scales, gradients and sweep mode of Hamming weights l_j on a ``Space`` of Categorical dimensions."""

    def __init__(self, space):
        bad = [d for d in space.dimensions if not isinstance(d, Categorical)]
        if bad:
            name = bad[0].name or f"dimension {space.dimensions.index(bad[0])}"
            raise ValueError(f"kernel='hamming' needs every dimension Categorical; {name} is {type(bad[0]).__name__}")
        self.n_dims = len(space.dimensions)
        self.n_categories = np.array([len(d.categories) for d in space.dimensions])
        widths = np.array([d.width for d in space.dimensions])
        self.col_dim = np.repeat(np.arange(self.n_dims), widths)           # dimension of each one-hot column
        self.col_factor = np.where(self.n_categories == 2, 2.0, 1.0)[self.col_dim]
        self.fixed_cols = np.flatnonzero(self.n_categories[self.col_dim] == 1)   # one-category columns: always 1, ℓ = 1

    def weights(self, l) -> np.ndarray:
        """l_j per dimension (a scalar is the isotropic l)."""
        return np.broadcast_to(np.asarray(l, dtype=np.float64), (self.n_dims,)).astype(np.float64)

    def length_scale(self, l) -> np.ndarray:
        """Per-column RBF length scales equal to Hamming weights l."""
        ls = (self.col_factor * self.weights(l)[self.col_dim]) ** -0.5
        ls[self.fixed_cols] = 1.0
        return ls

    def candidates(self, U):
        """Sampled candidates (NumPy array or torch tensor, one-hot rows) with every one-category column set to 1, as
        ``Categorical.to_unit`` encodes the told rows; modified in place and returned."""
        if len(self.fixed_cols):
            U[:, self.fixed_cols.tolist()] = 1
        return U

    def grad(self, g_cols) -> np.ndarray:
        """∂/∂log l_j from the per-column ∂/∂log ℓ_c."""
        g = -0.5 * np.bincount(self.col_dim, weights=np.asarray(g_cols, dtype=np.float64), minlength=self.n_dims)
        g[self.n_categories == 1] = 0.0          # their ℓ_c does not depend on l_j
        return g

    def kernel_argument(self, l) -> float:
        """S = Σ l_j over the dimensions that can differ: the kernel argument between two points that differ everywhere."""
        return float(self.weights(l)[self.n_categories >= 2].sum())

    def var_mode(self, l, requested: str) -> str:
        """The engine's var_mode for weights l: "auto" leaves the tensor cores only inside TC_RANGE."""
        if requested != "auto":
            return requested
        lo, hi = TC_RANGE
        return "auto" if lo <= self.kernel_argument(l) <= hi else "f64"
