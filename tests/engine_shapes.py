"""A host restatement of how the two persistent engines (csrc/engine.cuh, csrc/engine_batch.cuh) cut a model into work, so a
test can say which code paths a model shape reaches on G SMs:

- eng_split (engine.cuh:115): CTA b of G owns panels [P*b // G, P*(b+1) // G) of a matrix with P = N / 8 panels;
- row tiles (engine.cuh:678, engine_batch.cuh:606): the CTA walks its panels PT at a time, PT = 16 STRICT / 8 FAST
  (EngCfg<KS>::kPT, engine.cuh:108); the FAST second chain (`on1`) holds panels 4..7 of a tile;
- eng_kt (api.cu:1523): the largest of 512 / 256 / 128 / 64 whose tile (most panels a CTA owns, at most PT, x kt x 16 B) fits
  a 32 KB ring stage, capped at K; a CTA runs ceil(K / kt) k-tiles per row tile, the last one K % kt long when that is not 0;
- eng_sdpa_smem (engine.cuh:128) against ENG_WORK (engine.cuh:99): the longest SequenceLength the engines accept
  (engine_probe, api.cu:1463; the batch engine shares the probe);
- the launch cap (api.cu:1665): one decode-engine launch runs at most 65000 // n_phases steps, and the 16-bit tags restart
  at 1 after a zero-fill when a launch would pass 65535 (api.cu:1669).

This covers the FMA-pipe forms only: the batch engine's tensor-core form (LNB_BATCH_TC=1) sizes its tiles differently."""
from __future__ import annotations

STAGE_BYTES = 32 * 1024          # EngCfg<KS>::kStage = ENG_RING / kNST
ENG_WORK = 84 * 1024
TAG_LIMIT = 65535
LAUNCH_TAGS = 65000


def wide_args(G: int) -> dict:
    """`wide`: 32 heads of 64 over 8 KV heads, and an FFN sized from G so that a CTA owns 7 or 8 panels of w1|w3 (FAST: two
    chains, the second one partial) and w2's K = ffn_dim leaves a short last k-tile.  At G = 132: ffn_dim 4112."""
    from lnb_b200 import synth
    return dict(synth.TINY, dim=1536, n_layers=2, n_heads=32, n_kv_heads=8, head_dim=64, ffn_dim=4 * (8 * G - 28),
                vocab_size=32768, max_seq_len=512)


def deep_args() -> dict:
    """`deep`: TINY with 32 layers, 161 phases per decode-engine step"""
    from lnb_b200 import synth
    return dict(synth.TINY, n_layers=32, max_seq_len=448)


def tie_base_row(i: int) -> int:
    """`ties`: LM-head row i is a copy of row (i // 2) % 64, so every logit is shared by rows 2k, 2k+1, and 128 rows apart"""
    return (i // 2) % 64


def eng_split(P: int, b: int, G: int) -> tuple[int, int]:
    return P * b // G, P * (b + 1) // G


def panels_per_tile(strict: bool) -> int:
    return 16 if strict else 8


def eng_kt(strict: bool, N: int, K: int, G: int) -> int:
    per = (N // 8 + G - 1) // G
    maxp = max(1, min(panels_per_tile(strict), per))
    kt = 512
    while kt > 64 and maxp * kt * 16 > STAGE_BYTES:
        kt >>= 1
    return min(kt, K)


def eng_sdpa_smem(T: int, hd: int, n_rep: int) -> int:
    return T * ((hd + 8) + hd) * 2 + n_rep * (T * 12 + hd * 4) + n_rep * 5 * 8 + 64


def max_seq_len(args: dict) -> int:
    """the longest SequenceLength whose in-engine attention fits the work area"""
    hd, n_rep = args["head_dim"], args["n_heads"] // args["n_kv_heads"]
    T = 1
    while eng_sdpa_smem(T + 1, hd, n_rep) <= ENG_WORK:
        T += 1
    return T


def projections(args: dict) -> dict[str, tuple[int, int]]:
    """name -> (N, K) of every engine GEMV, single GPU"""
    q, kv = args["n_heads"] * args["head_dim"], args["n_kv_heads"] * args["head_dim"]
    d, f = args["dim"], args["ffn_dim"]
    return {"wqkv": (q + 2 * kv, d), "wo": (d, q), "w13": (2 * f, d), "w2": (d, f), "head": (args["vocab_size"], d)}


def row_tiles(P: int, b: int, G: int, strict: bool) -> list[tuple[int, int]]:
    """(first panel, np) of each row tile of CTA b"""
    p0, p1 = eng_split(P, b, G)
    PT = panels_per_tile(strict)
    return [(rt, min(PT, p1 - rt)) for rt in range(p0, p1, PT)]


def gemv_shape(N: int, K: int, G: int, strict: bool) -> dict:
    P = N // 8
    kt = eng_kt(strict, N, K, G)
    per_cta = [eng_split(P, b, G)[1] - eng_split(P, b, G)[0] for b in range(G)]
    tiles = [row_tiles(P, b, G, strict) for b in range(G)]
    return dict(panels=(min(per_cta), max(per_cta)),
                row_tiles=max(len(t) for t in tiles),
                nps=sorted({np_ for t in tiles for _, np_ in t}),
                kt=kt, k_tiles=(K + kt - 1) // kt, tail=K % kt,
                tiles_per_cta=[len(t) * ((K + kt - 1) // kt) for t in tiles])


def model_shape(args: dict, G: int, strict: bool) -> dict[str, dict]:
    return {name: gemv_shape(N, K, G, strict) for name, (N, K) in projections(args).items()}


def k_tiles_per_step(args: dict, G: int, strict: bool) -> tuple[float, int]:
    """(mean over the CTAs, max) of the k-tiles one consumer thread of each CTA waits for in one batch-engine step -- the
    `tiles` counter of engine_profile(batch=True)"""
    sh = model_shape(args, G, strict)
    per = [0] * G
    for name, s in sh.items():
        reps = 1 if name == "head" else args["n_layers"]
        for b in range(G):
            per[b] += reps * s["tiles_per_cta"][b]
    return sum(per) / G, max(per)


def n_phases(args: dict) -> int:
    """phases of one decode-engine step (api.cu engine_build, single GPU): qkv, attention, wo, w1|w3, w2 per layer + LM head"""
    return 5 * args["n_layers"] + 1


def engine_launches(n_steps: int, phases: int, tag: int) -> tuple[list[tuple[int, bool]], int]:
    """how engine_launch splits n_steps from next free tag `tag` (0: never launched): [(steps, tags wrapped first)], next tag"""
    cap = max(1, LAUNCH_TAGS // max(1, phases))
    out, done = [], 0
    while done < n_steps:
        n = min(n_steps - done, cap)
        wrap = tag == 0 or tag + n * phases > TAG_LIMIT
        if wrap:
            tag = 1
        out.append((n, wrap))
        tag += n * phases
        done += n
    return out, tag


def check_coverage(G: int) -> None:
    """the fixtures of test_gpu_engine.py reach every engine path this module names, on G SMs"""
    from lnb_b200 import synth
    wide, deep, t128 = wide_args(G), deep_args(), dict(synth.TINY128)
    for strict in (True, False):
        PT = panels_per_tile(strict)
        sh = model_shape(wide, G, strict)
        head, w13, w2, qkv = sh["head"], sh["w13"], sh["w2"], sh["wqkv"]
        # LM head: several row tiles per CTA (the batch engine's re-fetch at rt > p0), one of them partial; several k-tiles
        assert head["row_tiles"] >= 2 and min(head["nps"]) < PT and head["k_tiles"] >= 2, head
        assert head["kt"] == (128 if strict else 256), head
        # w1|w3: FAST's second chain (panels 4..7 of a tile) runs full and partial; STRICT eng_chain_tile<8> over several k-tiles
        if strict:
            assert w13["kt"] == 256 and w13["k_tiles"] >= 2, w13
        else:
            assert 8 in w13["nps"] and any(4 < p < 8 for p in w13["nps"]), w13
        # w2: K % kt != 0; the tail's 16 / 8 chunks are none of 64 / 32 / 16 / 8 (the STRICT generic chunk loop)
        assert w2["k_tiles"] >= 2 and w2["tail"] and (w2["tail"] // 8) not in (64, 32, 16, 8), w2
        # wq|wk|wv: eng_chain_tile<16> across k-tile boundaries
        assert qkv["kt"] == 512 and qkv["k_tiles"] >= 2, qkv
    # batch attention at n = 8: CTAs serve several (head, sequence) items
    assert wide["n_heads"] * 8 > G
    # engine position limits; the tag wrap of a 435-step run from the state a probe step leaves
    assert (max_seq_len(wide), max_seq_len(deep), max_seq_len(t128)) == (264, 444, 145)
    assert n_phases(deep) == 161 and LAUNCH_TAGS // n_phases(deep) == 403
    _, tag = engine_launches(1, n_phases(deep), 0)
    assert engine_launches(435, n_phases(deep), tag)[0] == [(403, False), (32, True)]
    # ties: the lowest row of every tie group has a partner in its panel and in another CTA, and (below row 120) in
    # another row tile of its own CTA
    V = wide["vocab_size"]
    groups = {}
    for i in range(V):
        groups.setdefault(tie_base_row(i), []).append(i)
    for strict in (True, False):
        for b, g in groups.items():
            kinds = tie_partner_kinds(g[0], g, V, G, strict)
            assert {"panel", "cta"} <= kinds, (b, kinds)
            if g[0] < 120:
                assert "tile" in kinds, (b, kinds)


def head_owner(row: int, vocab: int, G: int, strict: bool) -> tuple[int, int]:
    """(CTA, row tile index within that CTA) that computes LM-head row `row`"""
    P, p = vocab // 8, row // 8
    b = ((p + 1) * G - 1) // P                   # the last CTA whose first panel is <= p
    p0, p1 = eng_split(P, b, G)
    assert p0 <= p < p1
    return b, (p - p0) // panels_per_tile(strict)


def tie_partner_kinds(row: int, group: list[int], vocab: int, G: int, strict: bool) -> set[str]:
    """which kinds of tie partner `row` has among `group` (the rows with the same logit): "panel" (same 8-row panel), "tile"
    (same CTA, another row tile), "cta" (another CTA)"""
    b, t = head_owner(row, vocab, G, strict)
    kinds = set()
    for j in group:
        if j == row:
            continue
        if j // 8 == row // 8:
            kinds.add("panel")
            continue
        bj, tj = head_owner(j, vocab, G, strict)
        kinds.add("cta" if bj != b else "tile" if tj != t else "same_tile")
    return kinds
