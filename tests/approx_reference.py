"""tree_method=approx restated on top of the oracle's Trainer (TEST INFRASTRUCTURE): the per-tree cuts of csrc/booster.cu
(train_round, DMatrix::rebin_from_hessian).

Before the trees of class k in a boosting round grow, the cuts are made again by the shared cut rule (cuts_reference.py) with
the class's hessian as the weights: h_k at the round's starting margins, sample weight included, taken before row sampling.
The P trees of a forest share them.  Objectives with a constant hessian (reg:squarederror, reg:absoluteerror,
reg:quantileerror) keep the matrix's sample-weighted cuts, so approx grows hist trees for them.

Every tree is grown as tests/forest_reference.py grows it (a Trainer of its own whose next tree is that tree), on the bins of
its class's cuts.  At P = 1 the forest layout is the single-tree layout (eta / 1 == eta, tree 0 draws the single-tree rows)."""
import numpy as np

from oracle import gbt_oracle as O

import forest_reference as FR

CONSTANT_HESSIAN = ("reg:squarederror", "reg:linear", "reg:absoluteerror", "reg:quantileerror")


def resketches(objective):
    """approx makes each tree's cuts from its hessian: every objective whose hessian is not constant"""
    return objective not in CONSTANT_HESSIAN


def tree_cuts(X, max_bin, h):
    """The cuts one tree grows on: the oracle's cuts with the tree's hessian as the weights (ptrs, vals, mins, has_missing)."""
    return O.make_cuts(X, max_bin, np.ascontiguousarray(h, np.float32))


class ApproxTrainer(FR.ForestTrainer):
    """One update() = one boosting round of K * P trees under tree_method=approx; tree_cuts[t] are the cuts tree t grew on."""

    def __init__(self, params, X, y, P=1, base_score=None, weights=None, device_grid=True):
        super().__init__(params, X, y, P, base_score=base_score, weights=weights, device_grid=device_grid)
        self.max_bin = int(params.get("max_bin", 256))
        self.own_cuts, self.own_bins = self.cuts, self.bins
        self.grad_params = dict(params)
        self.tree_cuts = []

    def update(self):
        pre = self.m.copy()
        K, P, r = self.K, self.P, len(self.indptr) - 1
        masks = [FR.row_mask(self.seed, r, j, self.n, self.subsample) for j in range(P)]
        resketch = resketches(self.params.get("objective", "reg:squarederror"))
        gp = O.gradient(self.grad_params, pre, self.y, self.sw) if resketch else None
        for k in range(K):
            if resketch:
                self.cuts = tree_cuts(self.X, self.max_bin, gp[:, k, 1])
                self.bins = O.bin_matrix(self.X, self.cuts[0], self.cuts[1])
            else:
                self.cuts, self.bins = self.own_cuts, self.own_bins
            for j in range(P):
                tree = self._grow(pre, len(self.trees), k, masks[j])
                self.trees.append(tree)
                self.tree_cuts.append(self.cuts)
                self.info.append(k)
                one = self.model(len(self.trees) - 1)
                self.m[:, k] = self.m[:, k] + FR.leaf_values(one, self.X, 0)
        self.indptr.append(len(self.trees))
