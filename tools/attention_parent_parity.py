"""Bit-for-bit comparison of the head-width-64 flash kernel and rowdot between this library and another build of
libb200_e2eft.so (e.g. one built from an earlier commit) on the same seeded inputs: every output and log-sum-exp
must be bitwise equal.

    python tools/attention_parent_parity.py --other-lib /path/to/libb200_e2eft.so --out /tmp/parity.json"""
import argparse
import ctypes
import json
import os
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--other-lib", required=True)
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "attention_parity.json"))
    a = ap.parse_args()
    from diffusion_e2e_ft_b200 import lib, ops
    mine = lib.load()
    other = ctypes.CDLL(os.path.abspath(a.other_lib))
    for name in ("b200_attention_d64", "b200_rowdot_heads", "b200_last_error_string"):
        res, args = lib._SIGS[name]
        getattr(other, name).restype = res
        getattr(other, name).argtypes = args
    P = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)
    st = ops._stream()
    results = []
    # (B, heads, Lq, Lk, kv_segments, fused, want_lse): the SD-2 UNet levels, joint attention, cross-attention over
    # 77 and 1 keys, ragged lengths
    cases = [(8, 5, 9216, 9216, 2, True, False), (8, 10, 2304, 2304, 1, True, True), (8, 20, 576, 77, 1, False, True),
             (2, 5, 300, 200, 1, False, True), (4, 10, 129, 1, 1, False, False), (2, 20, 1, 127, 2, True, True)]
    for i, (B, heads, Lq, Lk, kvs, fused, want_lse) in enumerate(cases):
        C = heads * 64
        g = torch.Generator(device="cuda").manual_seed(100 + i)
        qkv = torch.randn(B, Lq, 3 * C, device="cuda", generator=g).half()
        kvb = qkv if (fused and Lk == Lq) else torch.randn(B, Lk, 3 * C, device="cuda", generator=g).half()
        q, k, v = qkv[..., :C], kvb[..., C:2 * C], kvb[..., 2 * C:]
        outs = []
        for L in (mine, other):
            o = torch.full((B, Lq, C), float("nan"), device="cuda", dtype=torch.float16)
            lse = torch.full((B, heads, Lq), float("nan"), device="cuda") if want_lse else None
            rc = L.b200_attention_d64(P(q), q.stride(0), q.stride(1), P(k), k.stride(0), k.stride(1), P(v), v.stride(0),
                                      v.stride(1), P(o), o.stride(0), o.stride(1), B, heads, Lq, Lk, kvs, 0.125 * 1.5,
                                      P(lse), st)
            assert rc == 0, L.b200_last_error_string()
            do = torch.randn(B, Lq, C, device="cuda", generator=torch.Generator(device="cuda").manual_seed(7)).half()
            d = torch.full((B, heads, Lq), float("nan"), device="cuda")
            rc = L.b200_rowdot_heads(P(do), do.stride(0), do.stride(1), P(o), o.stride(0), o.stride(1), B, Lq, heads,
                                     P(d), st)
            assert rc == 0, L.b200_last_error_string()
            torch.cuda.synchronize()
            outs.append((o, lse, d))
        (o1, l1, d1), (o2, l2, d2) = outs
        bits = lambda x, y: x is None or torch.equal(x.view(torch.int16 if x.dtype == torch.float16 else torch.int32),
                                                     y.view(torch.int16 if y.dtype == torch.float16 else torch.int32))
        r = dict(B=B, heads=heads, Lq=Lq, Lk=Lk, kv_segments=kvs, lse=want_lse, out_bitwise=bits(o1, o2),
                 lse_bitwise=bits(l1, l2), rowdot_bitwise=bits(d1, d2), finite=bool(torch.isfinite(o1).all()))
        print(json.dumps(r), flush=True)
        results.append(r)
    ok = all(r["out_bitwise"] and r["lse_bitwise"] and r["rowdot_bitwise"] and r["finite"] for r in results)
    with open(a.out, "w") as f:
        json.dump(dict(all_bitwise_equal=ok, cases=results), f, indent=1)
    print(json.dumps(dict(all_bitwise_equal=ok)))
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
