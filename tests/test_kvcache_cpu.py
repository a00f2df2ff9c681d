"""The MXFP8 KV cache without a GPU (DESIGN.md §9j): the C statement of its block rule (orc_kv_mxfp8_quantize in
oracle_sampling/lnb_sample_ref.c) against an integer restatement on the bf16 bit fields, and the reference forward with
quantized caches that the GPU tests compare against (RefSession), checked against orc_forward."""
import numpy as np
import pytest

import lnb_b200 as L
from oracle import oracle as O
from oracle_sampling import sample_ref as SR
from tests import mx_cases as MC
from tests.helpers import host_tensors, oracle_model
from tests.test_mxfp8_cpu import _e4m3, restate_dequant


# ---- the integer restatement of the block rule ------------------------------------------------------------------------
def _finite(b: int) -> bool:
    return (b & 0x7F80) != 0x7F80


def restate_kv(rows, head_dim, clamp_lo=-117, half_up=False):
    """codes, scales [n, n_kv, nb] and decoded bits of K or V rows [n, n_kv * head_dim], from integers alone (the
    decoded bits only for the rule's clamp: below it a code's value need not be a bf16 number)"""
    rows = np.asarray(rows, np.uint16)
    n, kv = rows.shape
    n_kv, nb = kv // head_dim, (head_dim + 31) // 32
    codes = np.zeros((n, kv), np.uint8)
    scales = np.zeros((n, n_kv, nb), np.uint8)
    deq = np.zeros((n, kv), np.uint16)
    for r in range(n):
        for h in range(n_kv):
            for b in range(nb):
                c0, c1 = h * head_dim + 32 * b, h * head_dim + min(32 * b + 32, head_dim)
                blk = [int(v) for v in rows[r, c0:c1]]
                mag = max([v & 0x7FFF for v in blk if _finite(v)] + [0])
                E = mag >> 7
                X = clamp_lo if E == 0 else max(clamp_lo, min(119, E - 127 - 8))
                scales[r, h, b] = (X + 127) & 0xFF
                for i, v in enumerate(blk):
                    if _finite(v):
                        c = _e4m3(v, X, half_up)
                        d = restate_dequant(c, X) if clamp_lo == -117 else 0
                    elif v & 0x7F:                     # NaN
                        c, d = 0x7F, 0x7FC0
                    else:                              # +-inf: saturated
                        c = ((v >> 8) & 0x80) | 0x7E
                        d = restate_dequant(c, X) if clamp_lo == -117 else 0
                    codes[r, c0 + i], deq[r, c0 + i] = c, d
    return codes, scales, deq


# ---- inputs: the MXFP8 weight cases laid out as head rows --------------------------------------------------------------
def case_rows(head_dim: int, n_kv: int = 2) -> np.ndarray:
    """the tie rows (X = -117, 0, 119), the edge rows (saturation, subnormals, the lower clamp, zero and -0 blocks) and the
    extreme blocks, cut into K/V rows of n_kv heads of head_dim (head_dim % 32 != 0: every head ends in a narrow block)"""
    src = [MC.mxfp8_tie_rows(), MC.mxfp8_edge_rows(), np.vstack(MC.mxfp8_extreme_blocks())]
    if head_dim % 32 == 0:
        flat = np.concatenate([a.reshape(-1) for a in src])      # whole 32-element blocks stay blocks
    else:                                                         # each 32-element case block starts a head
        heads = []
        for a in src:
            for row in a.reshape(-1, 32):
                heads.append(np.concatenate([row, row[:head_dim - 32]]) if head_dim > 32 else row[:head_dim])
        flat = np.concatenate(heads)
    w = n_kv * head_dim
    flat = np.concatenate([flat, np.zeros((-len(flat)) % w, np.uint16)])
    return flat.reshape(-1, w).astype(np.uint16)


def non_finite_rows(head_dim: int) -> np.ndarray:
    """blocks with NaN, +inf and -inf among finite values (the finite maximum sets X), and a block of only non-finite"""
    rng = np.random.default_rng(5)
    r = MC.bf16_trunc(rng.standard_normal((4, 2 * head_dim)).astype(np.float32))
    r[0, 3], r[0, 5], r[0, 9] = 0x7FC0, 0x7F80, 0xFF80          # NaN, +inf, -inf
    r[1, 0], r[1, 1] = 0x7F81, 0xFFC0                             # NaNs of other payloads and sign
    r[2, :32] = 0x7F80
    r[3, head_dim:] = 0xFF80
    return np.ascontiguousarray(r, np.uint16)


HEAD_DIMS = (32, 40, 48, 56, 64, 96, 128)


@pytest.mark.parametrize("hd", HEAD_DIMS)
def test_c_statement_matches_integer_restatement(hd):
    for rows in (case_rows(hd), non_finite_rows(hd)):
        c, s, d = SR.kv_mxfp8_quantize(rows, hd)
        rc, rs, rd = restate_kv(rows, hd)
        assert np.array_equal(s, rs)
        assert np.array_equal(c, rc), np.argwhere(c != rc)[:8]
        assert np.array_equal(d, rd), np.argwhere(d != rd)[:8]


def test_cases_cover_what_they_claim():
    c, s, _ = SR.kv_mxfp8_quantize(case_rows(32), 32)
    X = s.astype(int) - 127
    assert {-117, 0, 119} <= set(X.reshape(-1).tolist())             # ties at both clamps and at 0
    assert (c & 0x7F == 0x7E).any() and ((c & 0x7F) < 8).any()        # saturation, subnormals
    for hd in (40, 48, 56):                                            # tail blocks of 8, 16 and 24
        assert hd % 32 in (8, 16, 24) and SR.kv_mxfp8_quantize(case_rows(hd), hd)[1].shape[2] == 2
    c, s, d = SR.kv_mxfp8_quantize(non_finite_rows(64), 64)
    assert c[0, 3] == 0x7F and d[0, 3] == 0x7FC0 and c[0, 5] == 0x7E and c[0, 9] == 0xFE
    assert s[2, 0, 0] == 10 and (c[2, :32] == 0x7E).all()              # only inf: X = -117, every element +448 * 2^X


def test_broken_rules_are_caught():
    ties, edges = case_rows(64), case_rows(32)
    c, _, _ = SR.kv_mxfp8_quantize(ties, 64)
    assert not np.array_equal(c, restate_kv(ties, 64, half_up=True)[0])
    _, s, _ = SR.kv_mxfp8_quantize(edges, 32)
    assert not np.array_equal(s, restate_kv(edges, 32, clamp_lo=-127)[1])


# ---- the reference forward with quantized caches ----------------------------------------------------------------------
class RefSession:
    """orc_forward_order's sequence of oracle ops, with every K and V row the forward stores replaced by its decoded MXFP8
    blocks when kv_mx: what an MXFP8-cache session must compute.  order: O.ORDER_REF (STRICT) or O.ORDER_FAST_STREAM (the
    FAST order of the kernel chain with streamed attention, which every row of an MXFP8 session takes).  decode: rows
    [n, kv_l], head_dim -> the decoded rows stored in their place (default: the C statement's)"""

    def __init__(self, args: dict, tensors: dict, seq_len: int, kv_mx: bool, order=O.ORDER_REF, decode=None):
        self.a, self.t, self.seq_len, self.kv_mx = args, tensors, seq_len, kv_mx
        self.decode = decode or (lambda rows, hd: SR.kv_mxfp8_quantize(rows, hd)[2])
        self.ks, self.parts, self.attn = order
        kvd = args["n_kv_heads"] * args["head_dim"]
        self.ck = [np.zeros((seq_len, kvd), np.uint16) for _ in range(args["n_layers"])]
        self.cv = [np.zeros((seq_len, kvd), np.uint16) for _ in range(args["n_layers"])]
        self.pre_k = [np.zeros((seq_len, kvd), np.uint16) for _ in range(args["n_layers"])]   # rows before quantization
        self.pre_v = [np.zeros((seq_len, kvd), np.uint16) for _ in range(args["n_layers"])]
        _, self.cis = O.rope_table(args["head_dim"], 2 * args["max_seq_len"], args["rope_theta"], bool(args["use_scaled_rope"]))

    def _lin(self, x, w):
        return O.linear_bf16(x, w) if self.ks == 1 else O.linear_order_bf16(x, w, self.ks)

    def _norm(self, x, w, eps):
        if self.parts == 1:
            return O.rmsnorm(x, w, eps)
        r = O.rms_scale_order(x, eps, self.parts)        # rmsnorm_parts: t(t(x * r) * w), f32 products
        n1 = O.bf16_bits((O.bf16_to_f32(x) * r[:, None]).astype(np.float32))
        return O.bf16_bits((O.bf16_to_f32(n1) * O.bf16_to_f32(w)[None, :]).astype(np.float32))

    def load_caches(self, ck, cv, n):
        """positions [0, n) of every layer's caches: [layers][seq_len, kv_l] bf16 bits (a session's own decoded rows)"""
        for l in range(self.a["n_layers"]):
            self.ck[l][:n], self.cv[l][:n] = ck[l][:n], cv[l][:n]

    def forward(self, tokens, start_pos: int) -> np.ndarray:
        """logits [S, vocab] f32 of every row"""
        a, t = self.a, self.t
        hd, nh, nkv, eps = a["head_dim"], a["n_heads"], a["n_kv_heads"], a["norm_eps"]
        tokens = np.asarray(tokens, np.int64)
        S, T = len(tokens), start_pos + len(tokens)
        x = np.ascontiguousarray(t["tok_embeddings.weight"][tokens])
        for l in range(a["n_layers"]):
            p = f"layers.{l}."
            xn = self._norm(x, t[p + "attention_norm.weight"], eps)
            q = self._lin(xn, t[p + "attention.wq.weight"])
            k = self._lin(xn, t[p + "attention.wk.weight"])
            v = self._lin(xn, t[p + "attention.wv.weight"])
            q2 = O.rope_apply(np.ascontiguousarray(q.reshape(S, nh, hd)), self.cis, start_pos)
            k2 = O.rope_apply(np.ascontiguousarray(k.reshape(S, nkv, hd)), self.cis, start_pos).reshape(S, nkv * hd)
            self.pre_k[l][start_pos:T], self.pre_v[l][start_pos:T] = k2, v
            if self.kv_mx:
                k2, v = self.decode(k2, hd), self.decode(v, hd)
            self.ck[l][start_pos:T], self.cv[l][start_pos:T] = k2, v
            ck, cv = self.ck[l].reshape(self.seq_len, nkv, hd), self.cv[l].reshape(self.seq_len, nkv, hd)
            if self.attn == O.ATTN_REF:
                o = O.attention(q2, ck, cv, T, S > 1, q_pos0=start_pos)
            else:
                o = O.attention_order(q2, ck, cv, T, S > 1, start_pos, self.attn)
            h1 = O.add_bf16(x, self._lin(o, t[p + "attention.wo.weight"]))
            xn = self._norm(h1, t[p + "ffn_norm.weight"], eps)
            g = O.silu_bf16(self._lin(xn, t[p + "feed_forward.w1.weight"]))
            g = O.mul_bf16(g, self._lin(xn, t[p + "feed_forward.w3.weight"]))
            x = O.add_bf16(h1, self._lin(g, t[p + "feed_forward.w2.weight"]))
        lg = self._lin(self._norm(x, t["norm.weight"], eps), t["output.weight"])
        return (lg.astype(np.uint32) << 16).view(np.float32)


def test_reference_forward_is_orc_forward_and_stores_quantized_rows():
    args = dict(L.synth.TINY)
    tensors = host_tensors(args, 11)
    om = oracle_model(args, tensors)
    try:
        os_ = om.new_session(32)
        plain, quant = RefSession(args, tensors, 32, False), RefSession(args, tensors, 32, True)
        for toks, pos in (([1, 50, 999, 7, 300, 12, 64], 0), ([5], 7), ([77], 8)):
            lo = os_.forward(np.array(toks, np.int32), pos)
            lp = plain.forward(toks, pos)
            assert np.array_equal(lo.view(np.uint32), lp.view(np.uint32))
            lq = quant.forward(toks, pos)
            assert np.isfinite(lq).all()
        for l in range(args["n_layers"]):
            ok, ov = os_.cache(l)
            assert np.array_equal(ok.reshape(32, -1), plain.ck[l]) and np.array_equal(ov.reshape(32, -1), plain.cv[l])
        # layer 0 does not depend on earlier attention: its stored rows are D(Q(.)) of orc_forward's rows
        ok, ov = os_.cache(0)
        hd = args["head_dim"]
        assert np.array_equal(quant.ck[0], SR.kv_mxfp8_quantize(ok.reshape(32, -1), hd)[2])
        assert np.array_equal(quant.cv[0], SR.kv_mxfp8_quantize(ov.reshape(32, -1), hd)[2])
        assert not np.array_equal(quant.ck[0][:9], ok.reshape(32, -1)[:9])
        os_.close()
    finally:
        om.close()


def test_reference_forward_in_the_fast_stream_order_is_orc_forward_order():
    args = dict(L.synth.TINY)
    tensors = host_tensors(args, 12)
    om = oracle_model(args, tensors)
    try:
        os_ = om.new_session(32)
        ref = RefSession(args, tensors, 32, False, order=O.ORDER_FAST_STREAM)
        for toks, pos in (([1, 50, 999, 7, 300, 12, 64], 0), ([5], 7), ([77], 8)):
            lo = os_.forward(np.array(toks, np.int32), pos, order=O.ORDER_FAST_STREAM)
            assert np.array_equal(lo.view(np.uint32), ref.forward(toks, pos).view(np.uint32))
        os_.close()
    finally:
        om.close()
