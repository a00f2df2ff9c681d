"""Logits rows and sampler parameters at real vocabulary sizes, where every device job splits a row into CTAs of 4096
logits (PEN_SLICE, GRM_SLICE, SMP_SLICE and LP_SLICE) and the last slice is partial.  Shared by tests/test_vocab_rows_cpu.py
(the statement against its restatement, the routing rule) and tests/test_gpu_vocab_pipeline.py (the device against the
statement).  Everything here is pure numpy: no GPU."""
import numpy as np

SLICE = 4096              # logits per CTA of every job (csrc/sample.cuh, penalty.cuh, grammar.cuh, logprob.cuh)
SMP_THREADS = 1024        # threads of a sampler CTA: the most candidates sample_split_kernel ranks
SMP_MERGE = 2048          # candidates the last CTA of sample_split_kernel merges
VOCABS = (4112, 32000, 32768, 128256)   # 2 slices with a 16-logit tail; Llama 2's 8 slices; 8 full slices; Llama 3's 32

DEVICE_NAN = np.array([0x7FFFFFFF], np.uint32).view(np.float32)[0]   # the NaN the device's arithmetic makes
POS_NAN = np.array([0x7FC00000], np.uint32).view(np.float32)[0]
NEG_NAN = np.array([0xFFC00000], np.uint32).view(np.float32)[0]       # the x86 default NaN
FLT_MAX = np.float32(np.finfo(np.float32).max)


def slices(V: int) -> int:
    return -(-V // SLICE)


def last_slice(V: int) -> range:
    return range((slices(V) - 1) * SLICE, V)


def split_k(T: float, K: int, V: int) -> int:
    """smp_split_k (csrc/sample.cuh): the candidate count of a row sample_split_kernel serves, 0 for sample_kernel's rows"""
    k = V if K == 0 or K >= V else K
    return k if np.float32(T) > 0 and k <= SMP_THREADS and k * slices(V) <= SMP_MERGE else 0


def k_edge(V: int) -> int:
    """the largest top_k sample_split_kernel serves at V"""
    return min(SMP_THREADS, SMP_MERGE // slices(V))


def slices_of(idx, V: int) -> set:
    return {int(i) // SLICE for i in np.asarray(idx).reshape(-1)}


def allowed(rng, V: int, m: int, where: str) -> np.ndarray:
    """m token ids: "spread" over the row (always one in slice 0 and one in the last, partial slice) or "tail" (the last m
    ids, packed into the last slice and spilling backwards over its edge when m is larger)"""
    if where == "tail":
        return np.arange(V - m, V)
    if m == 1:
        return np.array([int(rng.choice(last_slice(V)))])
    idx = {int(rng.integers(0, SLICE)), int(rng.choice(last_slice(V)))}
    while len(idx) < m:
        idx.add(int(rng.integers(0, V)))
    return np.array(sorted(idx))


def masked_counts(V: int) -> list:
    """the allowed-token counts of the masked rows: 1, 2 and K - 1, K, K + 1 at K = 40 and at the split kernel's edge"""
    e = k_edge(V)
    return sorted({1, 2, 39, 40, 41, e - 1, e, e + 1})


def rows(rng, V: int) -> dict:
    """name -> f32 row [V]: the classes of test_sampling_cpu._rows, then the classes a sampler meets after a grammar mask, a
    -inf bias or a broken model, placed across the slice edges"""
    from tests.test_sampling_cpu import _rows
    out = dict(_rows(rng, V))
    base = rng.normal(0.0, 2.0, V).astype(np.float32)
    ninf = np.float32(-np.inf)
    for m in masked_counts(V):
        for where in ("spread", "tail"):
            r = np.full(V, ninf, np.float32)
            idx = allowed(rng, V, m, where)
            r[idx] = base[idx]
            out[f"masked_{where}_{m}"] = r
    z = np.full(V, ninf, np.float32)                      # a stuck grammar state: only two stop tokens, in the last slice
    lo = last_slice(V).start
    z[[lo + (V - lo) // 2, V - 1]] = [np.float32(-3.5), np.float32(-2.0)]
    out["z_only"] = z
    edges = base.copy()                                   # the same top value on both sides of every slice edge
    top = np.float32(base.max() + 1.0)
    for e in range(SLICE, V, SLICE):
        edges[e - 2:e + 2] = top
    edges[V - 1] = top
    out["edge_ties"] = edges
    zeros = -np.abs(base) - np.float32(1.0)               # +0.0 and -0.0 at the top, tied in value, not in rank
    zi = allowed(rng, V, 96, "spread")
    zeros[zi[::2]] = np.float32(0.0)
    zeros[zi[1::2]] = np.float32(-0.0)
    out["signed_zeros"] = zeros
    for name, v, at in (("pos_inf", np.float32(np.inf), V - 1), ("pos_nan", POS_NAN, SLICE),
                        ("device_nan", DEVICE_NAN, SLICE - 1), ("device_nan_0", DEVICE_NAN, 0)):
        r = base.copy()
        r[at] = v
        out[name] = r
    r = base.copy()
    r[rng.choice(V, V // 5, replace=False)] = NEG_NAN     # negative NaNs rank below everything
    out["neg_nan"] = r
    big = (np.sign(base) * (FLT_MAX - np.abs(rng.normal(0, 1e31, V)).astype(np.float32))).astype(np.float32)
    big[rng.choice(V, 5, replace=False)] = FLT_MAX        # l - m overflows to -inf below the top ties
    out["near_flt_max"] = big
    biased = base.copy()
    biased[rng.choice(V, V // 3, replace=False)] = ninf   # a -inf logit bias over a third of the row
    biased[V - 1] = ninf
    out["ninf_biased"] = biased
    return out


def ks(V: int) -> list:
    """top_k values: whole row, 1, 2, 40, both sides of the split kernel's edge, V - 1, V"""
    e = k_edge(V)
    return sorted({0, 1, 2, 40, e, e + 1, V - 1, V})


def cases(rng, V: int, row_dict: dict | None = None) -> list:
    """(name, row, (T, K, P, seed), p_next): every row with every K of ks(V), the temperature (0: greedy) and top-p cycling"""
    row_dict = rows(rng, V) if row_dict is None else row_dict
    Ts, Ps = (0.7, 1.0, 1e-3, 5.0, 0.0), (1.0, 0.9, 0.5, 1e-6)
    out, j = [], 0
    for name, r in row_dict.items():
        for K in ks(V):
            T, P = Ts[j % len(Ts)], Ps[(j // 3) % len(Ps)]
            out.append((name, r, (T, K, P, int(rng.integers(0, 2**63))), int(rng.integers(1, 10**6))))
            j += 1
    return out


def interleaved(case_list: list, n: int = 8) -> list:
    """the cases in launches of n rows, each launch holding rows of both sampler kernels while both kinds last"""
    split = [c for c in case_list if split_k(c[2][0], c[2][1], len(c[1]))]
    full = [c for c in case_list if not split_k(c[2][0], c[2][1], len(c[1]))]
    out = []
    while split or full:
        a = split[:n // 2]
        b = full[:n - len(a)]
        a = split[:n - len(b)]
        split, full = split[len(a):], full[len(b):]
        out.append(a + b)
    return out
