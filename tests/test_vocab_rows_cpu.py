"""The row classes and sampler parameters of tests/vocab_rows.py, without a GPU: at every real vocabulary size they reach
both sampler kernels on both sides of the split kernel's edge, the masked rows have their finite logits where they claim,
and the sampler's C statement (SR.sample_row) equals the independent restatement of test_sampling_cpu on them, so the
device is compared with a statement that is itself pinned on these rows."""
import numpy as np
import pytest

from oracle_sampling import sample_ref as SR
from tests import vocab_rows as VR
from tests.test_sampling_cpu import restated


def test_split_rule_restates_the_kernel_choice():
    # smp_split_k: k <= 1024 and k * slices <= 2048, for T > 0; K = 0 and K >= V mean the whole row
    assert [VR.k_edge(V) for V in VR.VOCABS] == [1024, 256, 256, 64]
    assert VR.split_k(0.7, 40, 128256) == 40 and VR.split_k(0.7, 64, 128256) == 64 and VR.split_k(0.7, 65, 128256) == 0
    assert VR.split_k(0.7, 256, 32000) == 256 and VR.split_k(0.7, 257, 32000) == 0
    assert VR.split_k(0.7, 1024, 4112) == 1024 and VR.split_k(0.7, 1025, 4112) == 0
    assert VR.split_k(0.0, 40, 32000) == 0 and VR.split_k(0.7, 0, 32000) == 0 and VR.split_k(0.7, 32000, 32000) == 0
    assert VR.split_k(0.7, 0, 1000) == 1000 and VR.split_k(0.7, 2000, 1000) == 1000   # one slice: the whole row splits


@pytest.mark.parametrize("V", VR.VOCABS)
def test_cases_reach_both_kernels_at_every_edge(V):
    rng = np.random.default_rng(V)
    cs = VR.cases(rng, V)
    e = VR.k_edge(V)
    params = [c[2] for c in cs]
    assert {1, e, e + 1, V - 1, V, 0} <= {K for _, K, _, _ in params}
    assert any(T == 0 for T, _, _, _ in params)
    for K, kernel in ((1, "split"), (2, "split"), (40, "split"), (e, "split"), (e + 1, "full"), (V - 1, "full"), (V, "full"),
                      (0, "full")):
        kinds = {("split" if VR.split_k(T, k, V) else "full") for T, k, _, _ in params if k == K and T > 0}
        assert kinds == {kernel}, (V, K, kinds)
    chunks = VR.interleaved(cs)
    assert sum(len(c) for c in chunks) == len(cs) and all(len(c) <= 8 for c in chunks)
    mixed = [c for c in chunks if len({bool(VR.split_k(x[2][0], x[2][1], V)) for x in c}) == 2]
    assert len(mixed) >= len(chunks) // 2, (len(mixed), len(chunks))


@pytest.mark.parametrize("V", VR.VOCABS)
def test_row_classes_sit_where_they_claim(V):
    rows = VR.rows(np.random.default_rng(V), V)
    last = VR.slices(V) - 1
    for name, r in rows.items():
        assert r.dtype == np.float32 and r.shape == (V,), name
        if name.startswith("masked_"):
            fin = np.flatnonzero(np.isfinite(r))
            m = int(name.rsplit("_", 1)[1])
            assert fin.size == m and last in VR.slices_of(fin, V), name
            if "spread" in name and m > 1:
                assert 0 in VR.slices_of(fin, V), name
    assert VR.slices_of(np.flatnonzero(np.isfinite(rows["z_only"])), V) == {last}
    u = rows["signed_zeros"].view(np.uint32)
    assert (u == 0).any() and (u == 0x80000000).any()
    assert (rows["device_nan"].view(np.uint32) == 0x7FFFFFFF).sum() == 1
    assert (rows["neg_nan"].view(np.uint32) == 0xFFC00000).any()
    top = rows["edge_ties"].max()
    for e in range(VR.SLICE, V, VR.SLICE):
        assert rows["edge_ties"][e - 1] == rows["edge_ties"][e] == top


@pytest.mark.parametrize("V,every", [(4112, 1), (32000, 4)])
def test_statement_equals_the_restatement_on_the_row_classes(V, every):
    rng = np.random.default_rng(V + 1)
    cs = VR.cases(rng, V)[::every]
    names = set()
    for name, row, (T, K, P, seed), pn in cs:
        want = restated(row, np.float32(T), K, P, seed, pn)
        assert SR.sample_row(row, T, K, P, seed, pn) == want, (V, name, T, K, P, seed, pn)
        names.add(name)
    assert {"z_only", "edge_ties", "signed_zeros", "device_nan", "near_flt_max", "ninf_biased"} <= names


def test_masked_rows_draw_only_allowed_tokens():
    for V in (32000, 128256):
        rng = np.random.default_rng(V + 2)
        for name, row in VR.rows(rng, V).items():
            if not (name.startswith("masked_") or name == "z_only"):
                continue
            for T, K, P in ((0.9, 40, 1.0), (0.9, 0, 0.9), (0.0, 0, 1.0), (1.0, VR.k_edge(V) + 1, 1.0)):
                t = SR.sample_row(row, T, K, P, 7, 100)
                assert np.isfinite(row[t]), (V, name, T, K, P, t)
