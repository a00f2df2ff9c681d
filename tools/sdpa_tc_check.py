"""sdpa_tc_kernel (tensor-core prompt attention, LNB_ACC_FAST) against the oracle's attention: distance statistics.
Usage: python tools/sdpa_tc_check.py [S ...]"""
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

import lnb_b200 as L
from oracle import oracle as O
from tests.helpers import bf16_ulp_diff, rand_bf16

c = L._capi
for S in [int(a) for a in sys.argv[1:]] or [70, 200, 513]:
    rng = np.random.default_rng(S)
    nh, nkv, hd = 32, 8, 128
    q = rand_bf16(rng, (S, nh, hd))
    ck, cv = rand_bf16(rng, (S, nkv, hd)), rand_bf16(rng, (S, nkv, hd))
    out = np.empty((S, nh * hd), np.uint16)
    t0 = time.time()
    exp = O.attention(q, ck, cv, S, 1)
    t1 = time.time()
    res = {}
    for tag, env in (("tc", "1"), ("fma", "0")):
        os.environ["LNB_SDPA_TC"] = env
        c.check(c.lib.lnb_op_attention_bf16(c.ptr(q, c.u16p), c.ptr(ck, c.u16p), c.ptr(cv, c.u16p), c.ptr(out, c.u16p), S, S, nh, nkv, hd, 1,
                                            c.LNB_ACC_FAST))
        d = bf16_ulp_diff(out, exp)
        a = np.abs(O.bf16_to_f32(out).astype(np.float64) - O.bf16_to_f32(exp).astype(np.float64))
        res[tag] = dict(max_ulp=int(d.max()), mismatch=float((out != exp).mean()), gt1=float((d > 1).mean()), max_abs=float(a.max()),
                        mean_abs=float(a.mean()))
    print(S, f"oracle {t1 - t0:.1f}s", res, flush=True)
