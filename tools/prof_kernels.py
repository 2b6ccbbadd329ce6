"""Tiny launcher for ncu captures of single kernels at production shapes.
    python tools/prof_kernels.py conv128|conv320|conv1280|attn|gn|linear
    python tools/prof_kernels.py vae [reps]   -- the VAE's hot convs as the model calls them (modules.py ResnetBlock2D /
                                                 Upsample2D, batch 8 at 768^2), each timed with the debug flags
                                                 0 (full), 16 (empty epilogue), 1 (no stores) and 8 (no MMAs)"""
import os, sys, math
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from diffusion_e2e_ft_b200 import ops
what = sys.argv[1]


def _vae_attribution(reps):
    L = ops._lib.load()
    g = torch.Generator(device="cpu").manual_seed(0)
    rnd = lambda *s, sc=1.0, dt=torch.float16: (torch.randn(*s, generator=g) * sc).to(dt).to("cuda")
    NB = 8
    cases = []     # (name, fn, flops)
    for H, C in ((768, 128), (384, 256), (192, 512)):
        x16 = rnd(NB, H, H, C)
        x32 = rnd(NB, H, H, C, dt=torch.float32)
        w = ops.pack_conv(rnd(C, C, 3, 3, sc=1 / math.sqrt(9 * C)))
        b = torch.zeros(C, device="cuda")
        fl = 2 * NB * H * H * C * 9 * C
        cases.append((f"conv1 {C}@{H} f16+stats", lambda x=x16, w=w, b=b, C=C: ops.conv2d(x, w, C, bias=b, stats=True), fl))
        cases.append((f"conv2 {C}@{H} f32+res+stats+f16copy",
                      lambda x=x16, w=w, b=b, C=C, r=x32: ops.conv2d(x, w, C, bias=b, residual=r, out_dtype=torch.float32,
                                                                      stats=True, f16_copy=True), fl))
    # shortcut conv2 (256 -> 128 at 768^2: decoder up-block 3, first resnet) and the 4-phase upsample (256 ch, 384 -> 768)
    xs = rnd(NB, 768, 768, 128); x2 = rnd(NB, 768, 768, 256)
    ws = ops.pack_conv(rnd(128, 128, 3, 3, sc=1 / math.sqrt(1152)), rnd(128, 256, 1, 1, sc=1 / 16))
    bs = torch.zeros(128, device="cuda")
    cases.append(("conv2 128@768 shortcut x2 f32+stats",
                  lambda: ops.conv2d(xs, ws, 128, bias=bs, x2=x2, out_dtype=torch.float32, stats=True, f16_copy=True),
                  2 * NB * 768 * 768 * 128 * (1152 + 256)))
    from diffusion_e2e_ft_b200.modules import Upsample2D
    up = Upsample2D(256).cuda()
    xu = rnd(NB, 384, 384, 256, dt=torch.float32)
    cases.append(("upsample 256@384->768 4-phase", lambda: up.run(xu, None, torch.float32),
                  2 * NB * 768 * 768 * 256 * 4 * 256))
    flags = (0, 16, 1, 8)
    print(f"{'shape':42s} " + " ".join(f"{'flag ' + str(f):>10s}" for f in flags) + "   TFLOP/s")
    with torch.no_grad():
        for name, fn, fl in cases:
            ms = []
            for f in flags:
                L.b200_debug_set_flags(f)
                try:
                    for _ in range(2):
                        fn()
                    torch.cuda.synchronize()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(reps):
                        fn()
                    e1.record(); torch.cuda.synchronize()
                finally:
                    L.b200_debug_set_flags(0)
                ms.append(e0.elapsed_time(e1) / reps)
            print(f"{name:42s} " + " ".join(f"{m:8.3f}ms" for m in ms) + f"   {fl / ms[0] / 1e9:7.1f}")


if what == "vae":
    if os.environ.get("B200_HALO"):      # 2: halo path even where the dispatcher calls the conv epilogue-bound
        ops._lib.load().b200_debug_set_halo(int(os.environ["B200_HALO"]))
    _vae_attribution(int(sys.argv[2]) if len(sys.argv) > 2 else 10)
    sys.exit(0)
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
from diffusion_e2e_ft_b200 import lib as _l
if len(sys.argv) > 3:
    _l.load().b200_debug_set_flags(int(sys.argv[3]))
if len(sys.argv) > 4:
    _l.load().b200_debug_force_block_n(int(sys.argv[4]))
if len(sys.argv) > 5:
    _l.load().b200_debug_set_swap(int(sys.argv[5]))
if os.environ.get("B200_HALO"):
    _l.load().b200_debug_set_halo(int(os.environ["B200_HALO"]))
dev = "cuda"
g = torch.Generator(device="cpu").manual_seed(0)
r = lambda *s, sc=1.0: (torch.randn(*s, generator=g) * sc).half().to(dev)
if what.startswith("conv"):
    cfg = {"conv128": (4, 768, 768, 128, 128), "conv128n8": (8, 768, 768, 128, 128), "conv128n2": (2, 768, 768, 128, 128), "conv256": (8, 384, 384, 256, 256), "conv512": (8, 192, 192, 512, 512),
           "conv320": (8, 96, 96, 320, 320), "conv640": (8, 48, 48, 640, 640), "conv1280": (8, 24, 24, 1280, 1280),
           "conv1280s": (8, 12, 12, 1280, 1280), "conv2560": (8, 24, 24, 2560, 1280)}[what]
    NB, H, W, Cin, Cout = cfg
    x = r(NB, H, W, Cin); w = ops.pack_conv(r(Cout, Cin, 3, 3, sc=1 / math.sqrt(9 * Cin))); b = torch.zeros(Cout, device=dev)
    st = True if os.environ.get("B200_STATS") else None
    fn = lambda: ops.conv2d(x, w, Cout, bias=b, stats=st)
    flops = 2 * NB * H * W * Cout * 9 * Cin
elif what.startswith("res"):          # res16 / res32: 128->128 768^2 conv with residual, fp16 / fp32 stream
    NB, H, W, Cin, Cout = 4, 768, 768, 128, 128
    odt = torch.float16 if what == "res16" else torch.float32
    x = r(NB, H, W, Cin); w = ops.pack_conv(r(Cout, Cin, 3, 3, sc=1 / math.sqrt(9 * Cin))); b = torch.zeros(Cout, device=dev)
    resid = r(NB, H, W, Cout).to(odt)
    fn = lambda: ops.conv2d(x, w, Cout, bias=b, residual=resid, out_dtype=odt)
    flops = 2 * NB * H * W * Cout * 9 * Cin
elif what == "attn2304":             # level-1 self-attention: 10 heads, 2304 tokens
    qkv = r(8, 2304, 1920)
    fn = lambda: ops.attention_d64(qkv[..., :640], qkv[..., 640:1280], qkv[..., 1280:], 10, 0.125)
    flops = 4 * 8 * 10 * 2304 * 2304 * 64
elif what == "attn":
    qkv = r(8, 9216, 960)
    fn = lambda: ops.attention_d64(qkv[..., :320], qkv[..., 320:640], qkv[..., 640:], 5, 0.125)
    flops = 4 * 8 * 5 * 9216 * 9216 * 64
elif what == "gn":
    x = r(4, 768, 768, 128); gm = torch.ones(128, device=dev); bt = torch.zeros(128, device=dev)
    fn = lambda: ops.group_norm(x, gm, bt, 1e-6)
    flops = 0
elif what == "gn32":                  # fp32 stream in, fp16 out: the VAE's dominant GroupNorm shape (6 B / element)
    x = r(4, 768, 768, 128).float(); gm = torch.ones(128, device=dev); bt = torch.zeros(128, device=dev)
    fn = lambda: ops.group_norm(x, gm, bt, 1e-6)
    flops = 0
elif what == "lin320":                # K = 320 GEMM with fp32 residual / output (attention out-proj, proj_out)
    a = r(73728, 320); w = r(320, 320, sc=0.05); b = torch.zeros(320, device=dev)
    resid = r(73728, 320).float()
    fn = lambda: ops.linear(a, w, b, residual=resid, out_dtype=torch.float32)
    flops = 2 * 73728 * 320 * 320
elif what.startswith("ln"):            # ln320 / ln640 / ln1280: the UNet's LayerNorms, fp32 stream in, fp16 out (6 B / element)
    C = int(what[2:]); rows = {320: 73728, 640: 18432, 1280: 4608}[C] * (8 if C != 320 else 1)
    x = r(rows, C).float(); gm = torch.ones(C, device=dev); bt = torch.zeros(C, device=dev)
    fn = lambda: ops.layer_norm(x, gm, bt)
    flops = 0; nbytes = rows * C * 6
elif what == "softmax":               # the VAE attention's score matrix of 2 images: fp32 in, fp16 out
    sm = r(2 * 9216, 9216).float()
    fn = lambda: ops.softmax_rows(sm, 0.044)
    flops = 0; nbytes = 2 * 9216 * 9216 * 6
elif what == "geglu":
    pass
elif what == "linear":
    a = r(73728, 320); w = r(2560, 320, sc=0.05); b = torch.zeros(2560, device=dev)
    fn = lambda: ops.linear(a, w, b)
    flops = 2 * 73728 * 320 * 2560
if what == "geglu":
    a = r(73728, 320); w0 = r(2560, 320, sc=0.05); b0 = torch.zeros(2560, device=dev)
    wg, bg = ops.pack_geglu(w0, b0)
    fn = lambda: ops.linear(a, wg, bg, act=ops.ACT_GEGLU)
    flops = 2 * 73728 * 320 * 2560
for _ in range(2):
    fn()
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(reps):
    fn()
e1.record(); torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / reps
print(f"{what}: {ms:.3f} ms/iter  {flops / ms / 1e9:.1f} TFLOP/s" + (f"  {nbytes / ms / 1e6:.0f} GB/s" if "nbytes" in dir() else ""))
