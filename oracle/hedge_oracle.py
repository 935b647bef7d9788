"""skopt's gp_hedge bookkeeping, restated for the tests (scikit-optimize ``optimizer/optimizer.py``: ``Optimizer.__init__``
with ``acq_func="gp_hedge"``, ``Optimizer._tell``, ``Optimizer.copy``) over the fixed-θ GP of ``gp_oracle``.

TEST INFRASTRUCTURE ONLY: nothing under ``kubeflow_b200/`` imports this module.

What skopt does, and what this class does:
* ``cand_acq_funcs_ = ["EI", "LCB", "PI"]``, ``gains_ = zeros(3)``, ``eta = 1.0``.
* ``_tell`` fits the model; if ``next_xs_`` exists, ``gains_ -= est.predict(vstack(next_xs_))`` — the NEW model's mean (raw
  y scale) at the previous picks.  Then, on one candidate set, each acquisition's first-index argmax becomes ``next_xs_``
  and the suggestion is ``next_xs_[argmax(rng.multinomial(1, softmax(eta · (gains_ − max gains_))))]``.
* ``copy()`` (what ``ask(n_points=k)`` works on) copies the gains; the copy has no ``next_xs_`` until its own first tell.
"""
from __future__ import annotations

import numpy as np

from . import gp_oracle as O

ACQS = (O.ACQ_EI, O.ACQ_LCB, O.ACQ_PI)


class HedgeOracle:
    def __init__(self, *, kind=O.KERNEL_MATERN52, length_scale=1.0, amplitude=1.0, noise=1e-3, xi=0.01, kappa=1.96, eta=1.0):
        self.theta = dict(kind=kind, length_scale=length_scale, amplitude=amplitude, noise=noise)
        self.xi, self.kappa, self.eta = xi, kappa, eta
        self.gains = np.zeros(len(ACQS))
        self.next_xs = None

    def copy(self):
        c = HedgeOracle(**self.theta, xi=self.xi, kappa=self.kappa, eta=self.eta)
        c.gains = self.gains.copy()
        return c

    def tell(self, Xt, y, cand, rng, update=True):
        """``_tell`` on the history (Xt transformed, y raw) with the candidate set ``cand``; ``update=False`` skips the gains
        update (the model is unchanged).  Returns (suggested row, per-acquisition first-index argmax, index drawn)."""
        fit = O.gp_fit(Xt, y, **self.theta)
        if update and self.next_xs is not None:
            self.gains = self.gains - O.gp_predict(fit, self.next_xs)[0]
        cand = np.asarray(cand, dtype=np.float64)
        mu, std = O.gp_predict(fit, cand)
        y_opt = float(np.min(fit["y"]))
        idx = [O.first_argmax(O.acquisition(mu, std, y_opt, a, self.xi, self.kappa)) for a in ACQS]
        self.next_xs = cand[idx]
        logits = self.gains - np.max(self.gains)
        e = np.exp(self.eta * logits)
        probs = e / np.sum(e)
        j = int(np.argmax(rng.multinomial(1, probs)))
        return self.next_xs[j], idx, j
