"""process_type=update (refresh and prune of existing trees) restated in NumPy, for the tests of csrc/refresh.cu.

Rules (DESIGN.md "Refresh and prune"; upstream TreeRefresher / TreePruner [UPSTREAM-RECALL]):
  * a row passes through a node when the predictor's walk on the raw float32 matrix does: x < split_cond goes left, a missing
    value follows default_left;
  * (g, h) are quantised on the round's fixed-point grid (max|g|, max h over every class -> power-of-two scales with
    grad_bits = 21 up to 2^20 rows, else 18), g_q = rint(g * sg), h_q = rint(h * sh) in float32, and summed exactly in int64;
  * G = g_q / sg, H = h_q / sh in double; sum_hess = float(H), base_weight = calc_weight(G, H), a split's
    loss_chg = (gain(L) + gain(R)) - gain(node) in float32; a leaf's base_weight is fl(eta / P) * w (w at the root), and with
    refresh_leaf its value is fl(eta / P) * w;
  * prune: every leaf in node order, TryPruneLeaf; the pruned tree is compacted in node order.
A model is the flat dict of the engine's export (left, right, parent, split_index, split_bin, default_left, split_cond, base_weight,
loss_chg, sum_hess, tree_offset, tree_info)."""
import numpy as np

FIELDS = ("left", "right", "parent", "split_index", "split_bin", "default_left", "split_cond", "base_weight", "loss_chg", "sum_hess")


def grad_bits_for(n):
    return 21 if n <= (1 << 20) else 18


def scales(g, h, n):
    """(sg, sh) of tree.cu scales_kernel from the round's pairs (every class)."""
    bits = grad_bits_for(n)
    mg = np.float32(np.max(np.abs(g))) if g.size else np.float32(0)
    mh = np.float32(np.max(h)) if h.size else np.float32(0)
    eg = int(np.frexp(mg)[1]) if mg > 0 and np.isfinite(mg) else 0
    eh = int(np.frexp(mh)[1]) if mh > 0 and np.isfinite(mh) else 0
    return np.float32(np.ldexp(1.0, bits - eg)), np.float32(np.ldexp(1.0, bits + 1 - eh))


def quantise(g, h, sg, sh):
    gq = np.rint(np.float32(g) * sg).astype(np.int64)
    hq = np.rint(np.float32(h) * sh).astype(np.int64)
    return gq, hq


class Param:
    def __init__(self, eta=0.3, lam=1.0, alpha=0.0, gamma=0.0, min_child_weight=1.0, max_delta_step=0.0, max_depth=6, P=1):
        self.eta = np.float32(np.float32(eta) / np.float32(P))
        self.lam, self.alpha = np.float32(lam), np.float32(alpha)
        self.gamma, self.mcw, self.mds = np.float32(gamma), np.float32(min_child_weight), np.float32(max_delta_step)
        self.max_depth = int(max_depth)


def _thr(w, alpha):
    return w - alpha if w > alpha else (w + alpha if w < -alpha else 0.0)


def calc_weight(p, G, H):
    if H < float(p.mcw) or H <= 0.0:
        return np.float32(0)
    dw = -_thr(G, float(p.alpha)) / (H + float(p.lam))
    if p.mds != 0 and abs(dw) > float(p.mds):
        dw = float(np.copysign(float(p.mds), dw))
    return np.float32(dw)


def calc_gain(p, G, H):
    if H <= 0.0:
        return np.float32(0)
    if p.mds == 0:
        t = _thr(G, float(p.alpha))
        return np.float32(t * t / (H + float(p.lam)))
    w = calc_weight(p, G, H)
    g, h = np.float32(G), np.float32(H)
    return -((np.float32(2) * g) * w + ((h + p.lam) * w) * w)


def tree_slice(model, t):
    a, b = int(model["tree_offset"][t]), int(model["tree_offset"][t + 1])
    return {k: np.array(model[k][a:b]) for k in FIELDS}


def leaf_of(tree, X):
    """The leaf each row of X reaches (the predictor's walk)."""
    n = X.shape[0]
    nid = np.zeros(n, np.int64)
    rows = np.arange(n)
    while True:
        internal = tree["left"][nid] != -1
        if not internal.any():
            return nid
        r = rows[internal]
        cur = nid[r]
        f = tree["split_index"][cur]
        v = X[r, np.minimum(f, X.shape[1] - 1)]
        v = np.where(f < X.shape[1], v, np.float32(np.nan))
        go_left = np.where(np.isnan(v), tree["default_left"][cur] != 0, v < tree["split_cond"][cur])
        nid[r] = np.where(go_left, tree["left"][cur], tree["right"][cur])


def node_sums(tree, X, gq, hq):
    """Exact int64 (G_q, H_q) of every node: the leaves over their rows, the reachable splits bottom-up (0 for unreachable slots)."""
    nn = len(tree["left"])
    G = np.zeros(nn, np.int64)
    H = np.zeros(nn, np.int64)
    leaf = leaf_of(tree, X)
    np.add.at(G, leaf, gq)
    np.add.at(H, leaf, hq)
    _, _, reach = _parents_depths(tree)
    for i in range(nn - 1, -1, -1):
        if reach[i] and tree["left"][i] != -1:
            G[i] = G[tree["left"][i]] + G[tree["right"][i]]
            H[i] = H[tree["left"][i]] + H[tree["right"][i]]
    return G, H


def refresh(tree, G, H, sg, sh, p, refresh_leaf, alive):
    isg, ish = 1.0 / float(sg), 1.0 / float(sh)
    for i in range(len(tree["left"])):
        if not alive[i]:
            continue
        g, h = float(G[i]) * isg, float(H[i]) * ish
        w = calc_weight(p, g, h)
        tree["sum_hess"][i] = np.float32(h)
        if tree["left"][i] == -1:
            tree["base_weight"][i] = w if i == 0 else p.eta * w
            if refresh_leaf:
                tree["split_cond"][i] = p.eta * w
        else:
            L, R = tree["left"][i], tree["right"][i]
            gl = calc_gain(p, float(G[L]) * isg, float(H[L]) * ish)
            gr = calc_gain(p, float(G[R]) * isg, float(H[R]) * ish)
            tree["base_weight"][i] = w
            tree["loss_chg"][i] = np.float32(gl + gr) - calc_gain(p, g, h)


def _parents_depths(tree):
    """Parents, depths and reachability from the root (children lie after their parent).  Slots no path reaches (upstream's
    deleted nodes) keep parent -1; the refresh leaves them out and the compaction drops them."""
    nn = len(tree["left"])
    par, depth, reach = np.full(nn, -1), np.zeros(nn, np.int64), np.zeros(nn, bool)
    reach[0] = True
    for i in range(nn):
        if reach[i] and tree["left"][i] != -1:
            for c in (tree["left"][i], tree["right"][i]):
                assert not reach[c], "a node with two parents"
                par[c], depth[c], reach[c] = i, depth[i] + 1, True
    return par, depth, reach


def prunable(tree, pid, depth_of_child, p):
    L, R = tree["left"][pid], tree["right"][pid]
    return (tree["left"][L] == -1 and tree["left"][R] == -1 and
            (tree["loss_chg"][pid] < p.gamma + np.float32(1e-6) or (p.max_depth > 0 and depth_of_child > p.max_depth)))


def make_leaf(tree, pid, p):
    tree["left"][pid] = -1
    tree["right"][pid] = -1
    tree["split_index"][pid] = 0
    tree["split_bin"][pid] = -1
    tree["default_left"][pid] = 0
    tree["loss_chg"][pid] = 0
    tree["split_cond"][pid] = p.eta * tree["base_weight"][pid]


def prune(tree, p, alive):
    par, depth, _ = _parents_depths(tree)
    for i in range(len(tree["left"])):
        if not alive[i] or tree["left"][i] != -1:
            continue
        cur, d = i, depth[i]
        while cur != 0:
            pid = par[cur]
            if not prunable(tree, pid, d, p):
                break
            alive[tree["left"][pid]] = alive[tree["right"][pid]] = False
            make_leaf(tree, pid, p)
            cur, d = pid, d - 1


def compact(tree, alive):
    par, _, _ = _parents_depths(tree)
    new = np.cumsum(alive) - 1
    out = {k: tree[k][alive].copy() for k in FIELDS}
    keep = np.nonzero(alive)[0]
    for j, i in enumerate(keep):
        for k in ("left", "right"):
            out[k][j] = -1 if tree[k][i] == -1 else new[tree[k][i]]
        out["parent"][j] = tree["parent"][0] if i == 0 else new[par[i]]
    return out


def update_tree(tree, X, gq, hq, sg, sh, p, ops, refresh_leaf):
    """One tree through the updaters `ops` ("refresh" / "prune"), in order; returns (tree, G_q, H_q) with the node sums of the
    input tree."""
    tree = {k: v.copy() for k, v in tree.items()}
    G, H = node_sums(tree, X, gq, hq)
    alive = _parents_depths(tree)[2]                   # unreachable slots are dead from the start
    for op in ops:
        if op == "refresh":
            refresh(tree, G, H, sg, sh, p, refresh_leaf, alive)
        else:
            prune(tree, p, alive)
    return compact(tree, alive), G, H


def predict_margin(trees, tree_info, X, K, base):
    """Float32 margins: base, then each tree's leaf added in model order (the predictor's sum)."""
    m = np.full((X.shape[0], K), np.float32(base), np.float32)
    for tr, k in zip(trees, tree_info):
        m[:, k] += tr["split_cond"][leaf_of(tr, X)]
    return m


def update_model(model, X, gradient, p, ops, refresh_leaf, K, P, base, rounds=None):
    """Refresh / prune every layer of `model` on X.  gradient(margin [n, K], round) -> float32 (n, K, 2) pairs.  Returns the
    updated trees (list of dicts), the node sums per tree and the per-round scales."""
    ntrees = len(model["tree_info"])
    per = K * P
    rounds = ntrees // per if rounds is None else rounds
    out, sums, scl = [], [], []
    info = [int(x) for x in model["tree_info"][: rounds * per]]
    for r in range(rounds):
        margin = predict_margin(out, info[: len(out)], X, K, base)
        gp = gradient(margin, r)
        sg, sh = scales(gp[:, :, 0], gp[:, :, 1], X.shape[0])
        scl.append((sg, sh))
        for t in range(r * per, (r + 1) * per):
            k = info[t]
            gq, hq = quantise(gp[:, k, 0], gp[:, k, 1], sg, sh)
            tr, G, H = update_tree(tree_slice(model, t), X, gq, hq, sg, sh, p, ops, refresh_leaf)
            out.append(tr)
            sums.append((G, H))
    return out, sums, scl


def flatten(trees):
    off = np.zeros(len(trees) + 1, np.int64)
    off[1:] = np.cumsum([len(t["left"]) for t in trees])
    return dict({k: np.concatenate([t[k] for t in trees]) for k in FIELDS}, tree_offset=off)
