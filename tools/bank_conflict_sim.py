#!/usr/bin/env python
"""How many shared-memory wavefronts does the decode table gather of one warp cost, for different table layouts?

The decode step's gather (`tab[x & 4095]`, 4-byte entries, 32 lanes with independent pseudo-random slots) is the
largest term of the LSU budget that bounds the round-1 word decode step (DESIGN.md section 6).  A wavefront serves one
4-byte word per bank (32 banks); lanes reading the SAME word are a broadcast.  The cost of one LDS is the largest
number of distinct words any bank has to deliver.  This Monte-Carlo compares candidate layouts; ncu
measured ~3.7 wavefronts per gather for the shipped layout (1 + 2.76 replays per step), the first row's 3.5 is the
same quantity in the model.

    python tools/bank_conflict_sim.py
"""
import numpy as np

TRIALS = 20000
rng = np.random.default_rng(7)


def wavefronts(word_addr):
    """word_addr: (trials, 32) word indices -> mean over trials of max distinct words per bank."""
    out = np.empty(word_addr.shape[0])
    for t, row in enumerate(word_addr):
        words = np.unique(row)
        out[t] = np.bincount(words % 32, minlength=32).max()
    return out.mean()


def slot_draws():
    """The decoder's slot is x mod 4096 of a well-mixed state: uniform over [0, 4096) whatever the model is
    (a skewed model only changes which SYMBOL a slot maps to), so one distribution covers every workload."""
    return rng.integers(0, 4096, (TRIALS, 32))


def main():
    lanes = np.arange(32)
    rows = []
    for kind in ("any model",):
        s = slot_draws()
        layouts = {
            "shipped: flat, 4 B per slot": s,
            "XOR swizzle (slot ^ (slot >> 5))": s ^ (s >> 5),
            "2 replicas, upper half-warp rotated by 16 banks": s + (lanes >= 16) * (4096 + 16),
            "4 replicas, quarter-warps rotated by 8 banks": s + (lanes // 8) * (4096 + 8),
            "2-byte entries (2 slots per word; needs a second gather)": s // 2,
            "1-byte slot->symbol table (4 slots per word; needs a second gather)": s // 4,
            "two half-warp loads (16 lanes each), summed": None,
            "bank-private replicas (32 x 16 KiB = 512 KiB: does not fit)": lanes + 32 * s,
        }
        for name, addr in layouts.items():
            if addr is None:
                w = wavefronts(s[:, :16]) + wavefronts(s[:, 16:])
            else:
                w = wavefronts(addr)
            rows.append((kind, name, w))
    width = max(len(r[1]) for r in rows)
    for kind, name, w in rows:
        print(f"{name:{width}s} {w:5.2f} wavefronts per gather")


if __name__ == "__main__":
    main()
