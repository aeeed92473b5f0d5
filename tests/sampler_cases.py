"""Weight sets of the key-sampler tests and the check of an alias table against its weights.

The sets are the shapes the apps use (Zipf^0.75 over a 10^6-word vocabulary for word2vec, degree^0.75 of an R-MAT graph
for node2vec) and the edges of the table builder: one to three keys, all weights equal, one weight 10^12 times the
others, zeros at the start, in the middle and at the end, and sizes that are and are not a power of two.
"""
import numpy as np

WEIGHT_SETS = ["n1", "n2", "n3", "equal", "equal-tenths", "huge", "zeros", "zipf-1m", "rmat-degree", "pow2", "not-pow2"]


def weights(name: str) -> np.ndarray:
    """float64 weights of set ``name``"""
    r = np.random.default_rng(WEIGHT_SETS.index(name))
    if name == "n1":
        return np.array([2.5])
    if name == "n2":
        return np.array([1.0, 3.0])
    if name == "n3":
        return np.array([0.2, 0.5, 0.3])
    if name == "equal":
        return np.ones(1000)
    if name == "equal-tenths":       # sum(w) rounds up, so every w n / sum is just below 1: all stay on the small stack
        return np.full(20, 0.1)
    if name == "huge":
        return np.concatenate([r.random(4000) + 0.5, [1e12 * 1.5], r.random(5999) + 0.5])
    if name == "zeros":
        w = r.random(5000) + 0.1
        w[:3] = 0; w[2400:2410] = 0; w[-4:] = 0
        return w
    if name == "zipf-1m":
        return (1.0 / np.arange(1, 10 ** 6 + 1)) ** 0.75
    if name == "rmat-degree":
        from adapm_b200.utils.graph import Graph, rmat_edges

        src, dst = rmat_edges(16, 8, seed=2)[:2]
        g = Graph.from_edges(src, dst, num_nodes=1 << 16)
        return g.degrees().cpu().numpy().astype(np.float64) ** 0.75      # isolated nodes: weight 0
    if name == "pow2":
        return r.random(1 << 16)
    if name == "not-pow2":
        return r.random((1 << 16) + 7)
    raise KeyError(name)


def table(w):
    """``(prob float32, alias int32)`` of the weights, from the extension's table builder"""
    from adapm_b200 import _C

    w = np.ascontiguousarray(w, dtype=np.float64)
    prob, alias = np.empty(w.size, dtype=np.float32), np.empty(w.size, dtype=np.int32)
    _C.build_alias_table(w.ctypes.data, w.size, prob.ctypes.data, alias.ctypes.data)
    return prob, alias


def table_errors(w, prob, alias):
    """Checks the table ``(prob, alias)`` of weights ``w`` and returns a list of what is wrong with it (empty: nothing).

    Form: ``prob`` in [0, 1], ``alias`` in [0, n), and a bucket that aliases to itself has ``prob == 1``: it keeps all its
    mass, which is what the builder gives the buckets left over when one stack runs empty.

    Zero weights: ``P_j == 0`` exactly, that is ``prob[j] == 0`` and no bucket aliases to ``j``.

    Distribution: with ``P = ops.alias_draw_probabilities(prob, alias)`` (table and device draw rule together) and
    ``p = w / sum(w)``, ``|P_j - p_j| <= T_j (2^-22 p_j + 2^-31)``, where ``T_j`` is the number of buckets that can draw
    ``j`` (its own and those that alias to it). Derivation: let ``q_i`` be the exact share of bucket ``i`` that stays
    on ``i`` in the float64 construction. Then ``p_j`` is the sum over those ``T_j`` buckets of ``(1/n)`` times ``q_j``
    (own) or ``1 - q_i`` (aliased). On the device, each bucket differs from that in three ways:
      - its share of the ``hi`` values is ``1/n`` within ``2^-32``;
      - ``prob`` is ``q`` rounded to float32, within ``2^-24 q``;
      - the share of ``lo`` below ``prob`` is ``prob`` within ``2^-24 prob + 2^-32``, because float32(lo) rounds ``lo``
        to 24 bits.
    So one bucket errs by at most ``2^-32 + (2^-23 q_i + 2^-32) / n``. That is ``<= 2^-23 p_j + 2^-31``:
      - ``q_j / n <= p_j`` for the own bucket;
      - for an aliased bucket, ``q_i / n <= 1/n <= p_j``, because only keys with ``w_j n / sum >= 1`` are ever aliased
        to.
    The float64 construction adds about ``(T_j + n) 2^-52 p_j``, which is below ``2^-23 p_j`` for ``n < 2^29``. The
    bound has a factor 2 on the ``p_j`` term for that. On the sets of this module the largest error is half the bound.
    """
    from adapm_b200.ops import alias_draw_probabilities

    w = np.asarray(w, dtype=np.float64)
    prob, alias = np.asarray(prob), np.asarray(alias).astype(np.int64)
    n = w.size
    errs = []
    own = np.arange(n)
    if prob.size != n or alias.size != n:
        return [f"table of {prob.size}/{alias.size} entries for {n} weights"]
    if not ((prob >= 0) & (prob <= 1)).all():
        errs.append(f"prob outside [0, 1] at {np.flatnonzero(~((prob >= 0) & (prob <= 1)))[:5]}")
    if not ((alias >= 0) & (alias < n)).all():
        return errs + [f"alias outside [0, {n}) at {np.flatnonzero(~((alias >= 0) & (alias < n)))[:5]}"]
    selfish = (alias == own) & (prob != 1)
    if selfish.any():
        errs.append(f"{int(selfish.sum())} buckets alias to themselves with prob != 1, e.g. {own[selfish][:5]}: "
                    f"{prob[selfish][:5]}")
    zero = w == 0
    if (prob[zero] != 0).any():
        errs.append(f"zero-weight keys with prob > 0: {own[zero & (prob != 0)][:5]}")
    to_zero = zero[alias] & (alias != own)
    if to_zero.any():
        errs.append(f"buckets alias to zero-weight keys: {own[to_zero][:5]} -> {alias[to_zero][:5]}")
    P = alias_draw_probabilities(prob, alias)
    if (P[zero] != 0).any():
        errs.append(f"zero-weight keys drawn with P > 0: {own[zero & (P != 0)][:5]}")
    p = w / w.sum()
    T = 1 + np.bincount(alias[alias != own], minlength=n)
    bound = T * (2.0 ** -22 * p + 2.0 ** -31)
    bad = np.abs(P - p) > bound
    if bad.any():
        j = own[bad][:5]
        errs.append(f"|P - w/W| over the bound at {j}: P {P[j]}, w/W {p[j]}, bound {bound[j]}")
    return errs
