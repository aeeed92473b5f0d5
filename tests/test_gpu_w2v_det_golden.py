"""The deterministic one-GPU word2vec steps (ops.sgns_step, ops.cbow_step, ops.hs_step) bit for bit against
tests/golden/w2v_det, made by running this file as a script. Each case runs three steps on a fresh seeded store and
records the SHA-256 of every row after them and the bits of each step's loss. The steps sum their updates in fixed
point, so the result does not depend on how the entries are grouped: any difference is a bug.

- SGNS at every VPL (d 16, 132, 300, 336) with 0, 5 and 30 negatives: Zipf keys, so each step has keys with more
  entries than one gather range, keys with one entry and repeated centres, and negatives equal to their pair's context.
- CBOW with 0 and 31 negatives and 1 and 32 context columns: padding, windows whose centre is < 0 and windows whose
  contexts are all padding.
- Hierarchical softmax with skip-gram (one context) and CBOW items, on trees whose longest path is 1 and 32.

    python tests/test_gpu_w2v_det_golden.py OUT_DIR    # writes OUT_DIR/golden.json"""
import hashlib
import json
import os
import struct
import sys

import numpy as np
import pytest
import torch

gpu = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "w2v_det", "golden.json")
ALPHA = 0.05
STEPS = 3

# (step, d or negatives, negatives or context columns or longest path)
CASES = ([("sgns", d, neg) for d in (16, 132, 300, 336) for neg in (0, 5, 30)]
         + [("cbow", neg, nc) for neg in (0, 31) for nc in (1, 32)]
         + [("hs", nc, n) for nc in (1, 10) for n in (1, 32)])


def _zipf(g, n_keys, shape):
    w = torch.arange(1, n_keys + 1, dtype=torch.float64) ** -1.05
    n = int(np.prod(shape))
    k = torch.multinomial(w, n, replacement=True, generator=g) if n else torch.zeros(0, dtype=torch.int64)
    return k.view(shape)


def _sgns_batch(g, n_keys, B, neg):
    k = _zipf(g, n_keys, (B, neg + 2))
    centers, contexts, negatives = k[:, 0].clone(), k[:, 1].clone(), k[:, 2:].contiguous()
    if neg:
        negatives[::5, 0] = contexts[::5]
    valid = negatives != contexts.view(-1, 1)
    cnt = torch.bincount(torch.cat([centers, contexts, negatives[valid]]), minlength=n_keys)
    assert (cnt > 64).any() and (cnt == 1).any() and centers.unique().numel() < B
    return centers, contexts, negatives


def _windows(g, vocab, B, nc, centres):
    """syn0 context keys [B, nc] (-1 = padding) for the given syn1 centres; some centres < 0, some windows all
    padding"""
    lens = torch.randint(0, nc + 1, (B,), generator=g)
    x = torch.where(torch.arange(nc).view(1, nc) < lens.view(B, 1), 2 * _zipf(g, vocab, (B, nc)), -1)
    x[:, 0] = 2 * _zipf(g, vocab, (B,))
    x[::17] = -1
    centres[5::23] = -1
    return centres, x


def _tree(n):
    from adapm_b200.utils.text import huffman_tree

    if n == 1:
        return huffman_tree([3, 5])
    fib = [1, 1]
    while len(fib) < n + 1:
        fib.append(fib[-1] + fib[-2])
    tree = huffman_tree(fib)
    assert tree.max_len == n
    return tree


def _case(kind, a, b):
    """(row width d, number of keys, a function that runs one step of a batch, the batches)"""
    from adapm_b200.ops import cbow_step, hs_step, sgns_step

    g = torch.Generator().manual_seed(1000 * len(kind) + 40 * a + b)
    if kind == "sgns":
        d, n_keys = a, 20000
        batches = [_sgns_batch(g, n_keys, 2048, b) for _ in range(STEPS)]
        return d, n_keys, lambda s, x, loss: sgns_step(s, *x, d, ALPHA, loss, impl="tma"), batches
    if kind == "cbow":
        d, vocab, B = 132, 8000, 2048
        batches = [_windows(g, vocab, B, b, 2 * _zipf(g, vocab, (B,)) + 1) + (2 * _zipf(g, vocab, (B, a)) + 1,)
                   for _ in range(STEPS)]
        return d, 2 * vocab, lambda s, x, loss: cbow_step(s, *x, d, ALPHA, loss, deterministic=True), batches
    tree, d, vocab, B = _tree(b), 300, 4000, 4096
    batches = [_windows(g, vocab, B, a, 2 * torch.randint(0, tree.num_words, (B,), generator=g) + 1)
               for _ in range(STEPS)]
    run = lambda s, x, loss: hs_step(s, *x, tree.to(s.device), d, ALPHA, loss, deterministic=True)  # noqa: E731
    return d, 2 * vocab, run, batches


def _name(case):
    return "{}_{}_{}".format(*case)


def _run(case):
    import adapm_b200 as ad

    d, n_keys, run, batches = _case(*case)
    name = _name(case)
    server = ad.Server(2 * d, num_keys=n_keys, num_threads=1, rank=0, world=1, backend="cuda", fabric="inproc",
                       job=f"w2vdet_{name}_{np.random.randint(1 << 30)}", device=0)
    kv = ad.Worker(0, server)
    try:
        g = torch.Generator().manual_seed(7)
        rows = torch.empty(n_keys, 2 * d)
        rows[:, :d] = torch.randn(n_keys, d, generator=g) * (0.5 / d ** 0.5)
        rows[:, d:] = torch.rand(n_keys, d, generator=g) * 0.1 + 1e-3
        allk = torch.arange(n_keys)
        kv.set(allk, rows.view(-1).clone())
        dev = server.device
        loss_bits = []
        for b in batches:
            loss = torch.zeros(1, device=dev)
            run(server, tuple(t.to(dev).contiguous() for t in b), loss)
            torch.cuda.synchronize()
            loss_bits.append(struct.pack("<f", float(loss.cpu()[0])).hex())
        got = torch.empty(n_keys * 2 * d)
        kv.pull(allk, got)
        return {"rows_sha256": hashlib.sha256(got.numpy().tobytes()).hexdigest(), "loss_bits": loss_bits}
    finally:
        kv.finalize()
        server.shutdown()


@gpu
@pytest.mark.parametrize("case", CASES, ids=_name)
def test_deterministic_steps_match_the_golden(case):
    with open(GOLDEN) as f:
        want = json.load(f)[_name(case)]
    assert _run(case) == want


if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    out = sys.argv[1]
    meta = {_name(case): _run(case) for case in CASES}
    os.makedirs(out, exist_ok=True)
    with open(os.path.join(out, "golden.json"), "w") as f:
        json.dump(meta, f, indent=1)
    print(json.dumps(meta))
