#!/usr/bin/env python
"""Record tests/golden/jpeg_symbols.npz: a few 8 x 8 blocks per quality whose frames code every Huffman symbol of
both tables -- DC categories 0-11 and all 162 AC symbols (runs 0-15 x sizes 1-10, EOB, ZRL), luma and chroma.

The blocks are chosen greedily from seeded candidates: 128 + a DC + one to three DCT basis functions with
log-uniform amplitudes, rounded and clipped.  oracle.jpeg.symbol_corpus_frames() lays them out as gray frames
(luma) and as RGB frames whose Cb is the block exactly (chroma), so a block's AC symbols do not depend on where it
sits.  After the AC symbols, blocks are appended whose DC differences reach the missing categories.  The result is
checked with oracle.jpeg.symbols() on the frames themselves.  Deterministic: a second run writes the same file.
"""
import io
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from oracle import jpeg as J  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "jpeg_symbols.npz")
QUALITIES = (100, 98, 95, 90, 75, 50)
CANDIDATES = 40000
SEED = 2024


def candidates(n, seed):
    """(n, 8, 8) uint8 blocks: 128 + DC + one to three basis functions (orthonormal DCT scale), rounded, clipped."""
    rng = np.random.default_rng(seed)
    x = np.arange(8)
    c = np.array([np.sqrt(0.125)] + [0.5] * 7)
    cos = c[:, None] * np.cos((2 * x[None] + 1) * np.arange(8)[:, None] * np.pi / 16)  # (u, x)
    basis = np.einsum("ux,vy->uvxy", cos, cos).reshape(64, 64)
    coef = np.zeros((n, 64))
    k = rng.integers(1, 4, n)
    pos = np.argsort(rng.random((n, 63)), 1)[:, :3] + 1
    amp = rng.normal(0, 1, (n, 3)) * 10 ** rng.uniform(0, 3, (n, 3))
    amp[np.arange(3)[None] >= k[:, None]] = 0
    np.put_along_axis(coef, pos, amp, 1)
    coef[:, 0] = rng.uniform(-1000, 1000, n)
    return np.clip(np.rint(128 + coef @ basis), 0, 255).astype(np.uint8).reshape(n, 8, 8)


def ac_symbols(coefs):
    """(n, 64) zig-zag coefficients -> (n, 256) bool: the AC symbols each block codes."""
    m = np.zeros((len(coefs), 256), bool)
    blk, k = np.nonzero(coefs[:, 1:])
    k = k + 1
    first = np.ones(len(blk), bool)
    first[1:] = blk[1:] != blk[:-1]
    run = k - np.where(first, 0, np.concatenate([[0], k[:-1]])) - 1
    m[blk, ((run & 15) << 4) | J._nbits(coefs[blk, k])] = True
    m[blk[run >= 16], 0xF0] = True
    last = np.zeros(len(coefs), np.int64)
    last[blk] = k
    m[last < 63, 0x00] = True
    return m


def cover_ac(cands, base):
    """Greedy: rarest uncovered symbol first, then the (quality, block) with it that covers the most -> {q: [i]}."""
    dcts = {q: J.fdct_quant(cands, J.quant_table(base, q)) for q in QUALITIES}
    has = np.concatenate([ac_symbols(dcts[q]) for q in QUALITIES])  # row qi * n + i
    want = np.zeros(256, bool)
    want[list(J.AC_SYMBOLS)] = True
    picks = {q: [] for q in QUALITIES}
    while True:
        open_ = want & has.any(0)
        if not open_.any():
            break
        counts = np.where(open_, has.sum(0), np.iinfo(np.int64).max)
        rows = np.nonzero(has[:, counts.argmin()])[0]
        row = rows[(has[rows] & open_).sum(1).argmax()]
        picks[QUALITIES[row // len(cands)]].append(int(row % len(cands)))
        want &= ~has[row]
    return picks, dcts


def extend_dc(picks, dcts, q):
    """Append blocks to quality q's list until its DC differences (from the predictor 0) reach every category."""
    dc = dcts[q][:, 0]
    seq = list(picks[q])
    for _ in range(64):
        prev = np.concatenate([[0], dc[seq][:-1]]) if seq else np.zeros(0, np.int64)
        got = set(J._nbits(dc[seq] - prev).tolist())
        missing = [c for c in J.DC_SYMBOLS if c not in got]
        if not missing:
            return seq
        last = dc[seq[-1]] if seq else 0
        cat = J._nbits(dc - last)
        hit = np.nonzero(cat == missing[-1])[0]
        # a category out of reach from here: step to the DC farthest away first
        seq.append(int(hit[0]) if len(hit) else int(np.abs(dc - last).argmax()))
    raise AssertionError(f"DC categories {missing} not reached")


def build():
    cands = candidates(CANDIDATES, SEED)
    corpus = {}
    for table, base in (("luma", J.LUMA_Q), ("chroma", J.CHROMA_Q)):
        picks, dcts = cover_ac(cands, base)
        picks[100] = extend_dc(picks, dcts, 100)
        for q, idx in picks.items():
            if idx:
                corpus[f"{table}_q{q}"] = cands[idx]
    return corpus


def coverage(corpus):
    """{(class, table, symbol)} the corpus frames code."""
    seen = set()
    for _, frame, q in J.symbol_corpus_frames(corpus):
        seen |= set(J.symbols(frame, q))
    return seen


def main():
    corpus = build()
    seen = coverage(corpus)
    for t, name in enumerate(("luma", "chroma")):
        dc = sorted(s for c, tt, s in seen if c == 0 and tt == t)
        ac = {s for c, tt, s in seen if c == 1 and tt == t}
        print(f"{name}: DC categories {dc}; AC symbols {len(ac)} of {len(J.AC_SYMBOLS)}, missing "
              f"{[(s >> 4, s & 15) for s in J.AC_SYMBOLS if s not in ac]}")
    buf = io.BytesIO()
    np.savez_compressed(buf, **{k: corpus[k] for k in sorted(corpus)})
    with open(OUT, "wb") as f:
        f.write(buf.getvalue())
    print("wrote", OUT, len(buf.getvalue()), "bytes,", {k: len(v) for k, v in sorted(corpus.items())})


if __name__ == "__main__":
    main()
