"""Gradient checkpointing of the VAE decoder (`B200AutoencoderKL.enable_gradient_checkpointing`: the `ckpt` mode of
autograd_blocks._ResnetFn and _VAEAttentionFn) on CPU with the kernels restated in torch (tests/cpu_emulation.py and
the d=512 restatements of test_vae_attention_bwd_cpu): the decoder's data gradient and the UNet gradients of both E2E
recipes are bitwise the same with it on and off, on the unfused and the memory-efficient attention and at an odd latent
size; the attention block's recompute gives its saved P / log-sum-exp; the switch and inference under no_grad.  The real kernels
run the same checks in test_vae_checkpointing_gpu.py."""
import numpy as np
import pytest
import torch

import cpu_emulation
import engine_checks as EC
import make_golden as MG
from diffusion_e2e_ft_b200 import autograd_blocks as ab
from diffusion_e2e_ft_b200 import ops
from oracle.unet import seeded_init
from oracle.vae import AutoencoderKLRef
from test_vae_attention_bwd_cpu import attention_d512, attention_d512_bwd, rowdot_d512

WIDE = (64, 128, 512)          # a decoder whose mid-block attention is 512 wide, so the d=512 kernels can take it


@pytest.fixture
def emulated(monkeypatch):
    cpu_emulation.install(monkeypatch)
    monkeypatch.setattr(ops, "FUSE_GN_STATS", False)
    for fn in (attention_d512, rowdot_d512, attention_d512_bwd):
        monkeypatch.setattr(ops, fn.__name__, fn)


def _vae(block_out_channels=None, memory_efficient=False):
    unet_ref, vae_ref = MG.build_tiny()
    if block_out_channels is not None:
        vae_ref = seeded_init(AutoencoderKLRef(MG.tiny_vae_config(block_out_channels=block_out_channels)), seed=77)
    _, vae = EC.engine_from_oracle(unet_ref, vae_ref.eval(), "cpu")
    if memory_efficient:
        vae.enable_xformers_memory_efficient_attention()
    return vae


def _nodes(t):
    """{block Function name: [saved is None, ...]} over the graph of t."""
    seen, stack, res = set(), [t.grad_fn], {}
    while stack:
        n = stack.pop()
        if n is None or n in seen:
            continue
        seen.add(n)
        if hasattr(n, "saved"):
            res.setdefault(type(n).__name__, []).append(n.saved is None)
        stack.extend(f for f, _ in n.next_functions)
    return res


def _decoder_dx(vae, z, dy, ckpt):
    if ckpt:
        vae.enable_gradient_checkpointing()
    else:
        vae.disable_gradient_checkpointing()
    ze = z.clone().requires_grad_(True)
    out = vae.decoder(ze)
    names = _nodes(out)
    out.backward(dy)
    return ze.grad, out.detach(), names


@pytest.mark.parametrize("wide,memory_efficient,hw", [
    (False, False, (8, 8)),            # the tiny config
    (False, False, (7, 5)),            # odd latent size
    (True, False, (6, 5)),             # 512-wide mid-block, unfused attention (saves P)
    (True, True, (6, 5)),              # 512-wide mid-block, d=512 flash attention (saves the LSE)
    (True, True, (5, 7)),
])
def test_decoder_dx_is_identical_with_checkpointing(emulated, wide, memory_efficient, hw):
    vae = _vae(WIDE if wide else None, memory_efficient)
    levels = len(vae.decoder.up_blocks)
    z = MG.inputs(4, 2, 4, *hw, scale=0.5)
    dy = MG.inputs(5, 2, 3, hw[0] << (levels - 1), hw[1] << (levels - 1))
    dx0, y0, names0 = _decoder_dx(vae, z, dy, False)
    dx1, y1, names1 = _decoder_dx(vae, z, dy, True)
    # checkpointed: every resnet and the attention block keep their inputs only; conv_in, the upsamplers and
    # conv_out keep what they saved
    assert names0 == {"_ConvInFnBackward": [False], "_ResnetFnBackward": [False] * (2 + 3 * levels),
                      "_VAEAttentionFnBackward": [False], "_UpsampleFnBackward": [False] * (levels - 1),
                      "_ConvOutFnBackward": [False]}, names0
    assert names1 == {"_ConvInFnBackward": [False], "_ResnetFnBackward": [True] * (2 + 3 * levels),
                      "_VAEAttentionFnBackward": [True], "_UpsampleFnBackward": [False] * (levels - 1),
                      "_ConvOutFnBackward": [False]}, names1
    assert torch.equal(y0, y1)
    assert torch.isfinite(dx0).all() and dx0.abs().max() > 0
    assert torch.equal(dx0, dx1)


@pytest.mark.parametrize("memory_efficient", [False, True])
def test_attention_recompute_gives_the_saved_tensors(emulated, memory_efficient):
    """The checkpointed attention block keeps x and its path; its recompute gives what the plain block saves: P on
    the unfused path, the log-sum-exp on the d=512 flash path."""
    from diffusion_e2e_ft_b200.vae import VAEAttention
    torch.manual_seed(0)
    att = VAEAttention(512, 32).eval().requires_grad_(False)
    with torch.no_grad():
        for p in att.parameters():
            p.normal_(0, 0.05)
    att.memory_efficient = memory_efficient
    x = torch.randn(2, 5, 6, 512, requires_grad=True)
    plain = ab.vae_attention(att, x).grad_fn
    ck = ab.vae_attention(att, x, ckpt=True).grad_fn
    assert ck.saved is None and ck.inputs[1] is x and ck.fused == memory_efficient
    again = ab._VAEAttentionFn.run(att, *ck.inputs)[1]
    assert len(again) == len(plain.saved) == 6 and (again[-1].dtype == torch.float32) == memory_efficient
    assert all(torch.equal(u, v) for u, v in zip(plain.saved, again))


def _unet_grads(unet):
    g = {n: p.grad.clone() for n, p in unet.named_parameters()}
    unet.zero_grad(set_to_none=True)
    return g


@pytest.mark.parametrize("recipe,noise_type", [("depth", "zeros"), ("normals", "gaussian"), ("geowizard", "zeros"),
                                               ("geowizard", "pyramid")])
def test_e2e_unet_gradients_are_identical_with_checkpointing(emulated, recipe, noise_type):
    """Both E2E recipes, zeros and noisy starts (vae.decode_from_prediction with the x_t addend)."""
    from diffusion_e2e_ft_b200 import DDIMScheduler
    from diffusion_e2e_ft_b200.training import LOSS_SCALE, e2e_ft_loss, e2e_ft_loss_geowizard
    unet_ref, vae_ref = MG.build_tiny("geowizard" if recipe == "geowizard" else "marigold")
    unet, vae = EC.engine_from_oracle(unet_ref, vae_ref, "cpu")
    unet.requires_grad_(True)
    g = torch.Generator().manual_seed(31)
    rgb = torch.rand(2, 3, 64, 64, generator=g) * 2 - 1
    mask = torch.rand(2, 1, 64, 64, generator=g) > 0.2
    depth = torch.rand(2, 1, 64, 64, generator=g) * 9.9 + 0.1
    normals = torch.nn.functional.normalize(torch.randn(2, 3, 64, 64, generator=g), dim=1)
    grads, losses = [], []
    for ckpt in (False, True):
        if ckpt:
            vae.enable_gradient_checkpointing()
        gen = torch.Generator().manual_seed(7)
        torch.manual_seed(7)                        # GeoWizard's pyramid noise draws from the global generators
        np.random.seed(7)
        if recipe == "geowizard":
            emb = MG.inputs(3, 2, 1, 96, scale=0.5)
            loss = e2e_ft_loss_geowizard(unet, vae, DDIMScheduler(), rgb, depth, normals, mask, emb,
                                         noise_type=noise_type, generator=gen)[0]
        else:
            gt = depth if recipe == "depth" else normals
            loss = e2e_ft_loss(unet, vae, DDIMScheduler(), rgb, gt, mask, MG.inputs(2, 1, 77, 128, scale=0.5),
                               recipe, noise_type=noise_type, generator=gen)[0]
        (loss * LOSS_SCALE).backward()
        losses.append(loss.detach())
        grads.append(_unet_grads(unet))
    assert torch.equal(losses[0], losses[1])
    assert any(g.abs().max() > 0 for g in grads[0].values())
    bad = [n for n in grads[0] if not torch.equal(grads[0][n], grads[1][n])]
    assert not bad, bad


def test_switch_and_inference(emulated):
    """diffusers' names: off by default, enable / disable toggle the decoder's segments; inference under no_grad is
    the same with the switch on, and the checkpointed training forward gives the inference bits."""
    vae = _vae()
    assert not vae.is_gradient_checkpointing and not vae.decoder.gradient_checkpointing
    z = MG.inputs(4, 2, 4, 6, 7, scale=0.5)
    with torch.no_grad():
        want = vae.decoder(z)
    vae.enable_gradient_checkpointing()
    assert vae.is_gradient_checkpointing and vae.decoder.gradient_checkpointing
    with torch.no_grad():
        got = vae.decoder(z)
        assert got.grad_fn is None and torch.equal(got, want)
    train = vae.decoder(z.clone().requires_grad_(True))
    assert all(_nodes(train)["_ResnetFnBackward"]) and torch.equal(train.detach(), want)
    vae.disable_gradient_checkpointing()
    assert not vae.is_gradient_checkpointing
    train = vae.decoder(z.clone().requires_grad_(True))
    assert not any(_nodes(train)["_ResnetFnBackward"]) and torch.equal(train.detach(), want)


# ------------------------------------------------------------------------------------------------ fused statistics
@pytest.fixture
def fused_stats(emulated, monkeypatch):
    """The fused GroupNorm statistics restated: a conv asked for `stats` accumulates the fp64 per-(image, channel) sum
    and sum of squares of what it writes and attaches them as `._cs`; group_norm_mean_rstd reads them when present
    (rounding differently from the statistics of the data).  Records which path each mean / rstd took."""
    monkeypatch.setattr(ops, "FUSE_GN_STATS", True)
    conv2d, mean_rstd, seen = ops.conv2d, ops.group_norm_mean_rstd, []

    def conv2d_stats(x, wp, cout, *a, stats=None, out_mul=1, out_off=(0, 0), **k):
        out = conv2d(x, wp, cout, *a, out_mul=out_mul, out_off=out_off, **k)
        if stats is not None and stats is not False:
            cs = torch.zeros(out.shape[0], cout, 2, dtype=torch.float64) if stats is True else stats
            part = out[:, out_off[0]::out_mul, out_off[1]::out_mul].double()
            cs[..., 0] += part.sum((1, 2))
            cs[..., 1] += part.pow(2).sum((1, 2))
            out._cs = cs
        return out

    def mean_rstd_cs(x1, eps, groups=32, x2=None):
        cs1, cs2 = getattr(x1, "_cs", None), getattr(x2, "_cs", None) if x2 is not None else None
        if cs1 is None or (x2 is not None and cs2 is None):
            seen.append(("data", tuple(x1.shape), id(x1)))
            return mean_rstd(x1, eps, groups, x2)
        seen.append(("cs", tuple(x1.shape), id(x1)))
        cs = cs1 if x2 is None else torch.cat([cs1, cs2], 1)
        NB, C = cs.shape[:2]
        g = cs.view(NB, groups, C // groups, 2).sum(2) / (x1.shape[1] * x1.shape[2] * (C // groups))
        var = (g[..., 1] - g[..., 0] ** 2).clamp_min(0)
        return torch.stack([g[..., 0], 1.0 / torch.sqrt(var + eps)], -1).float().contiguous()
    monkeypatch.setattr(ops, "conv2d", conv2d_stats)
    monkeypatch.setattr(ops, "group_norm_mean_rstd", mean_rstd_cs)
    return seen


def test_recompute_reads_the_fused_statistics_of_the_kept_inputs(fused_stats):
    """With the fused statistics, a checkpointed block's recompute reads the `_cs` its kept input carries, as the plain
    forward did: the mean / rstd take the same path and give the same bits, and so does dx."""
    vae = _vae()
    z = MG.inputs(4, 2, 4, 8, 8, scale=0.5)
    dy = MG.inputs(5, 2, 3, 64, 64)
    dx0, _, _ = _decoder_dx(vae, z, dy, False)
    plain = list(fused_stats)
    fused_stats.clear()
    dx1, _, _ = _decoder_dx(vae, z, dy, True)
    # the checkpointed forward takes the plain one's paths; each recompute in its backward takes, for a block input,
    # the path the forward took on that same (kept) tensor object
    fwd, rec = fused_stats[:len(plain)], fused_stats[len(plain):]
    assert [f[:2] for f in fwd] == [p[:2] for p in plain]
    path_of = {i: path for path, _, i in fwd}
    kept = [(path, path_of[i]) for path, _, i in rec if i in path_of]
    assert kept and sum(path == "cs" for path, _ in kept) > 0 and all(a == b for a, b in kept), kept
    assert torch.equal(dx0, dx1)
