"""The engines' work split restated on the host (tests/engine_shapes.py): at 132 SMs (H100 SXM) the fixtures of
test_gpu_engine.py reach the engine paths TINY never does, and the restatement agrees with hand-computed values."""
from tests import engine_shapes as ES


def test_fixtures_reach_every_engine_path_at_132_sms():
    ES.check_coverage(132)


def test_restatement_at_132_sms():
    G = 132
    wide = ES.wide_args(G)
    assert wide["ffn_dim"] == 4112
    strict, fast = ES.model_shape(wide, G, True), ES.model_shape(wide, G, False)
    # LM head: 4096 panels over 132 CTAs; STRICT tiles of 16 + 15 / 16 at kt 128, FAST 4 tiles of 7 / 8 at kt 256
    assert strict["head"]["panels"] == (31, 32) and strict["head"]["nps"] == [15, 16] and strict["head"]["k_tiles"] == 12
    assert fast["head"]["row_tiles"] == 4 and fast["head"]["nps"] == [7, 8] and fast["head"]["k_tiles"] == 6
    assert strict["w13"]["panels"] == (7, 8) and fast["w13"]["nps"] == [7, 8] and fast["w13"]["kt"] == 256
    assert strict["w2"]["panels"] == (1, 2) and strict["w2"]["kt"] == 512 and strict["w2"]["k_tiles"] == 9
    assert strict["w2"]["tail"] == 16
    assert strict["wqkv"]["panels"] == (2, 3) and strict["wqkv"]["k_tiles"] == 3
    # one 8-sequence session has twice as many attention items as CTAs
    assert wide["n_heads"] * 8 == 256
    # a CTA's row tiles cover exactly its panels
    for b in (0, 1, 77, 131):
        p0, p1 = ES.eng_split(4096, b, G)
        assert sum(n for _, n in ES.row_tiles(4096, b, G, True)) == p1 - p0
    assert ES.eng_split(4096, 131, G)[1] == 4096
