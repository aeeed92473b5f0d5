"""The device key sampler's alias tables, input checks and numpy replay, without a GPU.

``ops.alias_draw_probabilities`` gives the exact distribution a table draws under the device rule, so the tables are
compared with ``w / sum(w)`` directly instead of through a histogram. ``ops.sample_keys_reference`` is checked here
against a per-draw Python loop; ``test_gpu_sampler.py`` checks the kernel against it bit for bit.
"""
import math

import numpy as np
import pytest
import torch

from multirank import one_rank_store
from sampler_cases import WEIGHT_SETS, table, table_errors, weights


@pytest.mark.parametrize("name", WEIGHT_SETS)
def test_alias_table_draws_the_weights(name):
    """Each table has the right form, never draws a zero-weight key, and draws ``w / W`` within the bound derived in
    ``sampler_cases.table_errors``."""
    w = weights(name)
    prob, alias = table(w)
    assert table_errors(w, prob, alias) == []
    if name in ("zeros", "rmat-degree"):
        assert (w == 0).sum() > 0
    if name == "equal-tenths":       # the buckets left over on the small stack: prob 1, alias itself
        assert (prob == 1).all() and (alias == np.arange(w.size)).all()


def test_table_check_sees_a_wrong_table():
    """The check fails on tables that are wrong by a little: one bucket's prob off by 2^-16 (a change of 2^-16 / n in
    the draw probability of two keys), one bucket aliased to a
    zero-weight key, a self-aliased bucket with prob 0.999."""
    w = weights("zeros")
    prob, alias = table(w)
    i = int(np.flatnonzero((prob > 0.25) & (prob < 0.75))[0])
    p2 = prob.copy(); p2[i] += 2.0 ** -16
    assert any("over the bound" in e for e in table_errors(w, p2, alias))
    a2 = alias.copy(); a2[i] = 0
    assert any("alias to zero-weight" in e for e in table_errors(w, prob, a2))
    w3 = weights("equal-tenths")
    p3, a3 = table(w3)
    p3[4] = 0.999
    assert any("alias to themselves" in e for e in table_errors(w3, p3, a3))


def test_alias_draw_probabilities_counts_buckets_and_lo_values():
    """Hand-counted cases: n = 3 splits the 2^32 hi values 1431655766 / 1431655765 / 1431655765; prob 0.5 keeps
    exactly 2^31 lo values (float32(lo) < 2^31 for lo < 2^31 - 64, and the 64 below round up to 2^31)."""
    from adapm_b200.ops import alias_draw_probabilities

    P = alias_draw_probabilities(np.ones(3, np.float32), np.arange(3))
    assert P.tolist() == [1431655766 / 2 ** 32, 1431655765 / 2 ** 32, 1431655765 / 2 ** 32]
    P = alias_draw_probabilities(np.array([0.5, 1.0], np.float32), np.array([1, 1]))
    assert P[0] == (2 ** 31 - 64) / 2 ** 33 and P[0] + P[1] == 1.0
    P = alias_draw_probabilities(np.array([0.0, 1.0], np.float32), np.array([1, 1]))
    assert P.tolist() == [0.0, 1.0]


BAD_WEIGHTS = {"negative": [1.0, -1.0, 2.0], "nan": [1.0, math.nan], "inf": [math.inf, 1.0], "-inf": [1.0, -math.inf],
               "empty": [], "all-zero": [0.0, 0.0, 0.0], "sum-overflows": [1.5e308, 1.5e308]}


@pytest.mark.parametrize("case", list(BAD_WEIGHTS))
def test_bad_weights_are_refused(case):
    """Negative weights gave prob < 0 (``[-1, 2]``: key 1 always) and infinite ones prob 0 for all others (``[inf, 1]``:
    key 0 always) without an error; now the table builder and DeviceSampler refuse them."""
    from adapm_b200 import AdapmError, _C
    from adapm_b200.ops import DeviceSampler

    w = torch.tensor(BAD_WEIGHTS[case], dtype=torch.float64)
    n = w.numel()
    prob, alias = torch.empty(max(n, 1), dtype=torch.float32), torch.empty(max(n, 1), dtype=torch.int32)
    with pytest.raises(AdapmError):
        _C.build_alias_table(w.data_ptr(), n, prob.data_ptr(), alias.data_ptr())
    with pytest.raises(AdapmError):
        _C.alias_distribution(w.data_ptr(), n, 0, 1)
    with one_rank_store(4, 16, "cpu", "float32") as (s, _):
        with pytest.raises(ValueError):
            DeviceSampler(s, weights=w)


def test_too_many_weights_are_refused():
    """The alias entries are int32: more than 2^31 - 1 weights are refused before any is read."""
    from adapm_b200 import AdapmError, _C
    from adapm_b200.ops import DeviceSampler

    buf = torch.ones(4, dtype=torch.float64)
    out_p, out_a = torch.empty(4, dtype=torch.float32), torch.empty(4, dtype=torch.int32)
    with pytest.raises(AdapmError, match="int32"):
        _C.build_alias_table(buf.data_ptr(), 1 << 31, out_p.data_ptr(), out_a.data_ptr())
    with one_rank_store(4, 16, "cpu", "float32") as (s, _):
        with pytest.raises(ValueError, match="2\\^31"):
            DeviceSampler(s, weights=torch.ones(1, dtype=torch.float64).expand(1 << 31))


@pytest.mark.parametrize("distribution", ["uniform", "log-uniform"])
@pytest.mark.parametrize("num_keys", [0, -3, 1 << 32, (1 << 32) + 5])
def test_key_counts_out_of_range_are_refused(distribution, num_keys):
    """``num_keys = 0`` drew ``first_key`` every time, and ``num_keys >= 2^32`` overflows the 64-bit ``hi * n``."""
    from adapm_b200.ops import DeviceSampler

    with one_rank_store(4, 16, "cpu", "float32") as (s, _):
        with pytest.raises(ValueError, match="num_keys"):
            DeviceSampler(s, distribution=distribution, num_keys=num_keys)
        DeviceSampler(s, distribution=distribution, num_keys=(1 << 32) - 1)
        DeviceSampler(s, distribution=distribution, num_keys=1)
        with pytest.raises(ValueError, match="distribution"):
            DeviceSampler(s, distribution="zipf", num_keys=10)


# ---------------------------------------------------------------------------------------------- reference vs brute force
M64 = (1 << 64) - 1


def _mix64(x):
    x ^= x >> 33; x = (x * 0xff51afd7ed558ccd) & M64
    x ^= x >> 33; x = (x * 0xc4ceb9fe1a85ec53) & M64
    return x ^ (x >> 33)


def _brute(n, seed, kind, prob, alias, num, first, stride, resident=None, max_tries=64):
    """one draw at a time, with Python integers and numpy float32 scalars"""
    keys, checks, misses = [], 0, 0
    for i in range(n):
        t = 0
        while True:
            h = _mix64((seed & M64) ^ ((i * 0x9E3779B97F4A7C15 + t * 0xD1B54A32D192ED03) & M64))
            hi, lo = h >> 32, h & 0xFFFFFFFF
            if kind == "alias":
                b = (hi * num) >> 32
                j = b if np.float32(lo) * np.float32(2.0 ** -32) < prob[b] else int(alias[b])
            elif kind == "uniform":
                j = (hi * num) >> 32
            else:
                j = min(max(int(math.floor(math.exp(hi * 2.0 ** -32 * math.log(num + 1)))) - 1, 0), num - 1)
            k = first + j * stride
            if resident is None:
                break
            checks += 1
            if resident[k]:
                break
            t += 1
            if t >= max_tries:
                misses += 1
                break
        keys.append(k)
    return np.array(keys, dtype=np.int64), checks, misses


@pytest.mark.parametrize("kind,num,first,stride", [("alias", 0, 1, 2), ("alias", 0, 0, 1), ("uniform", 7, 100, 3),
                                                   ("uniform", 1, 5, 1), ("log-uniform", 50, 17, 1),
                                                   ("log-uniform", 1, 0, 2)])
@pytest.mark.parametrize("seed", [3, 0xF00D_0000_0000_0001, -1])
def test_reference_matches_per_draw_loop(kind, num, first, stride, seed):
    from adapm_b200.ops import sample_keys_reference

    w = np.array([0.5, 0.0, 3.0, 1.0, 0.25])
    prob, alias = table(w)
    num = w.size if kind == "alias" else num
    n = 700
    got = sample_keys_reference(n, seed, distribution=kind, prob=prob, alias=alias, num_keys=num, first_key=first,
                                key_stride=stride, chunk=256)
    want, _, _ = _brute(n, seed, kind, prob, alias, num, first, stride)
    assert got.tolist() == want.tolist()
    if kind == "alias":
        assert 1 * stride + first not in set(got.tolist())          # the zero-weight key
    resident = np.zeros(first + num * stride + 1, dtype=bool)
    resident[first + stride * np.arange(0, num, 2)] = True          # every second key
    for max_tries in (1, 2, 64):
        got = sample_keys_reference(n, seed, distribution=kind, prob=prob, alias=alias, num_keys=num, first_key=first,
                                    key_stride=stride, resident=resident, max_tries=max_tries, chunk=256)
        want = _brute(n, seed, kind, prob, alias, num, first, stride, resident, max_tries)
        assert (got[0].tolist(), got[1], got[2]) == (want[0].tolist(), want[1], want[2]), max_tries

