"""The NumPy split reference (tests/split_reference.py) against the oracle's own split enumeration (oracle/gbt_oracle.c
eval_split_mono), on the same dequantised histograms: the unconstrained best split must agree bit for bit.  Runs on the CPU."""
import itertools

import numpy as np
import pytest

import split_reference as R

f32 = np.float32


def _oracle_best(oracle, params, hist, tot, cuts, scales):
    cut_ptrs, cut_vals, min_vals = cuts
    F = len(cut_ptrs) - 1
    flat = np.concatenate([hist[f, :cut_ptrs[f + 1] - cut_ptrs[f]] for f in range(F)]).astype(np.float64)
    flat[:, 0] *= float(scales[2]); flat[:, 1] *= float(scales[3])
    G, H = tot[0] * float(scales[2]), tot[1] * float(scales[3])
    p = R.Params.of(params)
    root_gain = R.calc_gain(p, G, H)[()]
    import ctypes as C
    assert np.float32(oracle.lib().orc_calc_gain(C.byref(oracle.make_params(params)), G, H)).view(np.uint32) == f32(root_gain).view(np.uint32)
    return oracle.eval_split(params, flat, cut_ptrs, cut_vals, min_vals, G, H, root_gain)


def _check(oracle, params, hist, tot, cuts, scales, has_missing):
    ref = R.eval_node(params, hist, cuts[0], cuts[1], cuts[2], has_missing, tot, scales)
    orc = _oracle_best(oracle, params, hist, tot, cuts, scales)
    best = ref["best"]
    if best is None:
        assert orc["split_bin"] == -1 and orc["loss_chg"] == 0
        return
    assert (orc["findex"], orc["split_bin"], orc["default_left"]) == (best["feature"], best["bin"], best["dleft"])
    assert f32(orc["loss_chg"]).view(np.uint32) == best["loss_chg"].view(np.uint32)
    if ref["expanded"]:
        assert f32(orc["split_value"]).view(np.uint32) == f32(ref["tree"]["split_cond"][0]).view(np.uint32)


PARAMS = [dict(reg_lambda=l, alpha=a, max_delta_step=m, min_child_weight=c)
          for l, a, m, c in itertools.product([0.0, 1.0, 10.0], [0.0, 0.5], [0.0, 0.7], [0.0, 1.0, 6.5])]


@pytest.mark.parametrize("missing", [0.0, 0.2])
@pytest.mark.parametrize("params", PARAMS, ids=lambda p: "l%g-a%g-m%g-c%g" % (p["reg_lambda"], p["alpha"], p["max_delta_step"], p["min_child_weight"]))
def test_reference_best_split_equals_the_oracle(oracle, params, missing):
    rng = np.random.default_rng(hash((params["reg_lambda"], params["alpha"], params["max_delta_step"], params["min_child_weight"], missing)) & 0xffff)
    for trial in range(3):
        F = int(rng.integers(1, 40))
        nb = rng.choice([1, 2, 8, 33, 255] + ([256] if missing == 0 else []), size=F)
        hist, tot, cuts = R.synth_node(rng, nb, n_rows=int(rng.integers(5, 300)), missing_frac=missing,
                                       gmax=int(rng.choice([3, 1 << 10, 1 << 21])), hmax=int(rng.choice([2, 1 << 12, 1 << 22])))
        scales = R.scales_for(f32(rng.uniform(0.1, 100)), f32(rng.uniform(0.1, 10)), 21)
        _check(oracle, params, hist, tot, cuts, scales, missing > 0)


@pytest.mark.parametrize("missing", [0.0, 0.3])
def test_reference_tie_rules_equal_the_oracle(oracle, missing):
    """Duplicated columns (equal candidates across features), empty bins (equal candidates inside a feature) and a tiny
    integer grid (many equal gains): lower feature, then earlier scan position, in both."""
    rng = np.random.default_rng(7)
    for trial in range(20):
        F = int(rng.integers(2, 12))
        nb = rng.choice([2, 4, 8], size=F)
        src = int(rng.integers(0, F - 1))
        dst = int(rng.integers(src + 1, F))
        nb[dst] = nb[src]
        hist, tot, cuts = R.synth_node(rng, nb, n_rows=int(rng.integers(3, 20)), missing_frac=missing, gmax=2, hmax=2, dup=[(src, dst)])
        scales = R.scales_for(f32(1), f32(1), 21)
        for params in (dict(reg_lambda=1.0, min_child_weight=0.0), dict(reg_lambda=0.0, max_delta_step=0.7, min_child_weight=0.0)):
            _check(oracle, params, hist, tot, cuts, scales, missing > 0)


def test_bynode_reference_keeps_the_smallest_draws():
    """The node subset has max(1, floor(frac * |parent|)) features, all inside the parent set."""
    parent = np.ones(4096, bool)
    m = R.bynode_mask(parent, 0.1, 3, 0, 0)
    assert m.sum() == 409
    parent[::3] = False
    assert R.bynode_mask(parent, 0.5, 3, 2, 5).sum() == int(np.floor(f32(0.5) * f32(parent.sum())))
    assert not (R.bynode_mask(parent, 0.5, 3, 2, 5) & ~parent).any()
