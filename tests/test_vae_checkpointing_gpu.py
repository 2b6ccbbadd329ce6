"""GPU tests of the VAE decoder's gradient checkpointing (`B200AutoencoderKL.enable_gradient_checkpointing`: the
`ckpt` mode of autograd_blocks._ResnetFn and _VAEAttentionFn): the recompute of every block reproduces the tensors a
plain training forward saves
bit for bit (fused GroupNorm statistics, fp16 twins, the unfused path's P, the d=512 path's log-sum-exp), at the tiny
config and at 768 x 768.  The forward is reproducible in practice but not by construction: the GroupNorm statistics
merge fp64 partial sums with atomics, and a different order could change the last bit of an fp32 mean / rstd; the decoder's data gradient and the UNet gradients of a Marigold and a GeoWizard E2E
micro-step equal the plain ones; at the recipe's shape (bs 2, 768 x 768) the checkpointed micro-step peaks lower; and a
2048 x 2048 micro-step on the memory-efficient attention completes with finite gradients when the device has room.

Bitwise gradients need a deterministic backward.  The GroupNorm backward and the loss reductions sum with fp32
atomics, whose order can change the last bits from one run to the next, so each gradient check also runs the plain
path twice: where those two agree bit for bit the checkpointed run must too, and otherwise it may differ from the plain
run by no more than the plain runs differ from each other."""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GB = 1024 ** 3
WIDE = (64, 128, 512)          # a tiny decoder whose mid-block attention is 512 wide (the d=512 kernels can take it)


def _tiny_vae(wide=False, memory_efficient=False):
    import engine_checks as EC
    import make_golden as MG
    from oracle.unet import seeded_init
    from oracle.vae import AutoencoderKLRef
    unet_ref, vae_ref = MG.build_tiny()
    if wide:
        vae_ref = seeded_init(AutoencoderKLRef(MG.tiny_vae_config(block_out_channels=WIDE)), seed=77).eval()
    _, vae = EC.engine_from_oracle(unet_ref, vae_ref, DEV)
    if memory_efficient:
        vae.enable_xformers_memory_efficient_attention()
    return vae


def _full_vae():
    from diffusion_e2e_ft_b200 import B200AutoencoderKL
    torch.manual_seed(1234)
    with torch.device(DEV):
        vae = B200AutoencoderKL()
    return vae.eval().requires_grad_(False)


# ------------------------------------------------------------------------------------------------ recompute bits
def _chain(out):
    """The decoder graph from its output back to z, one node per block: a chain, since every block has one input."""
    nodes, n = [], out.grad_fn
    while n is not None and type(n).__name__ != "AccumulateGrad":
        nodes.append(n)
        nxt = [f for f, _ in n.next_functions if f is not None]
        n = nxt[0] if nxt else None
    return nodes


def _flat(saved):
    out = []
    for t in saved:
        if isinstance(t, (list, tuple)):
            out += _flat(t)
        elif torch.is_tensor(t):
            out.append(t)
    return out


def _saved_per_block(out):
    """(block, recomputed?, saved tensors) of every block Function in the graph of `out`; a checkpointed block is
    re-run as its backward re-runs it (its Function's `run` on the inputs it kept)."""
    from diffusion_e2e_ft_b200 import autograd_blocks as ab
    fns = {"_ResnetFnBackward": ab._ResnetFn, "_VAEAttentionFnBackward": ab._VAEAttentionFn}
    res = []
    for n in _chain(out):
        name = type(n).__name__
        if getattr(n, "saved", 0) is None:
            res.append((name, True, _flat(fns[name].run(n.m, *n.inputs)[1])))
        elif hasattr(n, "saved"):
            res.append((name, False, _flat(n.saved)))
    return res


def _check_recompute(vae, z):
    vae.disable_gradient_checkpointing()
    plain = _saved_per_block(vae.decoder(z.clone().requires_grad_(True)))
    vae.enable_gradient_checkpointing()
    ck = _saved_per_block(vae.decoder(z.clone().requires_grad_(True)))
    vae.disable_gradient_checkpointing()
    torch.cuda.synchronize()
    assert [n for n, _, _ in plain] == [n for n, _, _ in ck]
    assert not any(r for _, r, _ in plain)
    assert {n for n, r, _ in ck if r} == {"_ResnetFnBackward", "_VAEAttentionFnBackward"}
    assert {n for n, r, _ in ck if not r} == {"_ConvInFnBackward", "_UpsampleFnBackward", "_ConvOutFnBackward"}
    for i, ((name, _, a), (_, _, b)) in enumerate(zip(plain, ck)):
        assert len(a) == len(b), (i, name)
        for j, (u, v) in enumerate(zip(a, b)):
            assert u.dtype == v.dtype and u.shape == v.shape and torch.equal(u, v), (i, name, j)
    return plain


@pytest.mark.parametrize("wide,memory_efficient", [(False, False), (True, False), (True, True)])
def test_recompute_equals_the_saved_forward_tiny(wide, memory_efficient):
    import make_golden as MG
    vae = _tiny_vae(wide, memory_efficient)
    saved = _check_recompute(vae, MG.inputs(4, 2, 4, 12, 10, scale=0.5).to(DEV))
    att = [s for n, _, s in saved if n == "_VAEAttentionFnBackward"][0]
    # unfused: x, mean/rstd, hn, qk, P, O; d=512 flash path: x, mean/rstd, hn, qkv, O, lse
    assert len(att) == 6 and (att[-1].dtype == torch.float32) == memory_efficient


def test_recompute_equals_the_saved_forward_768():
    """SD VAE widths, bs 2, 96 x 96 latents (768 x 768 images), the default (unfused) mid-block attention."""
    vae = _full_vae()
    g = torch.Generator(device="cpu").manual_seed(8)
    _check_recompute(vae, (torch.randn(2, 4, 96, 96, generator=g) * 0.5).to(DEV))


# ------------------------------------------------------------------------------------------------ gradients
def _equal_or_within_rerun_spread(plain, plain2, ck, what):
    """ck equals plain bit for bit when the plain backward reproduces itself; else it is as close to plain as a plain
    rerun is (the order of fp32 atomics is the only difference left)."""
    assert plain.keys() == plain2.keys() == ck.keys()
    same, worst_rerun, worst_ck = True, 0.0, 0.0
    for k in plain:
        a, a2, b = plain[k].float(), plain2[k].float(), ck[k].float()
        same = same and torch.equal(plain[k], plain2[k])
        scale = a.abs().max().item() or 1.0
        worst_rerun = max(worst_rerun, (a2 - a).abs().max().item() / scale)
        worst_ck = max(worst_ck, (b - a).abs().max().item() / scale)
    bitwise = all(torch.equal(plain[k], ck[k]) for k in plain)
    print(f"{what}: plain reruns bitwise {same} (max rel {worst_rerun:.2e}); checkpointed bitwise {bitwise} "
          f"(max rel {worst_ck:.2e})")
    if same:
        assert bitwise, what
    else:
        assert worst_ck <= max(2 * worst_rerun, 1e-6), (what, worst_ck, worst_rerun)


def _decoder_dx(vae, z, dy, ckpt):
    (vae.enable_gradient_checkpointing if ckpt else vae.disable_gradient_checkpointing)()
    ze = z.clone().requires_grad_(True)
    vae.decoder(ze).backward(dy)
    torch.cuda.synchronize()
    vae.disable_gradient_checkpointing()
    return {"dx": ze.grad}


@pytest.mark.parametrize("config", ["tiny", "tiny_512_memory_efficient", "768"])
def test_decoder_dx_with_checkpointing(config):
    import make_golden as MG
    if config == "768":
        vae, shape = _full_vae(), (2, 4, 96, 96)
    else:
        vae, shape = _tiny_vae(config != "tiny", config != "tiny"), (2, 4, 12, 10)
    up = 2 ** (len(vae.decoder.up_blocks) - 1)
    g = torch.Generator(device="cpu").manual_seed(9)
    z = (torch.randn(*shape, generator=g) * 0.5).to(DEV)
    dy = torch.randn(shape[0], 3, shape[2] * up, shape[3] * up, generator=g).to(DEV)
    plain, plain2, ck = (_decoder_dx(vae, z, dy, c) for c in (False, False, True))
    assert torch.isfinite(ck["dx"]).all() and ck["dx"].abs().max() > 0
    _equal_or_within_rerun_spread(plain, plain2, ck, f"decoder dx {config}")


def _e2e_grads(kind, ckpt):
    """One tiny E2E micro-step (Marigold depth or GeoWizard depth + normals) with the decoder checkpointed or not."""
    import engine_checks as EC
    import make_golden as MG
    from diffusion_e2e_ft_b200 import DDIMScheduler
    from diffusion_e2e_ft_b200.training import LOSS_SCALE, e2e_ft_loss, e2e_ft_loss_geowizard
    unet_ref, vae_ref = MG.build_tiny(kind)
    unet, vae = EC.engine_from_oracle(unet_ref, vae_ref, DEV)
    unet.requires_grad_(True)
    if ckpt:
        vae.enable_gradient_checkpointing()
    g = torch.Generator().manual_seed(23)
    rgb = (torch.rand(2, 3, 64, 64, generator=g) * 2 - 1).to(DEV)
    mask = (torch.rand(2, 1, 64, 64, generator=g) > 0.2).to(DEV)
    depth = (torch.rand(2, 1, 64, 64, generator=g) * 9.9 + 0.1).to(DEV)
    if kind == "geowizard":
        normals = torch.nn.functional.normalize(torch.randn(2, 3, 64, 64, generator=g), dim=1).to(DEV)
        emb = (torch.randn(2, 1, 96, generator=g) * 0.5).to(DEV)
        loss = e2e_ft_loss_geowizard(unet, vae, DDIMScheduler(), rgb, depth, normals, mask, emb)[0]
    else:
        ctx = (torch.randn(1, 77, 128, generator=g) * 0.5).to(DEV)
        loss = e2e_ft_loss(unet, vae, DDIMScheduler(), rgb, depth, mask, ctx, "depth")[0]
    (loss * LOSS_SCALE).backward()
    torch.cuda.synchronize()
    return {n: p.grad for n, p in unet.named_parameters() if p.grad is not None}


def _e2e_unet_params(kind):
    import make_golden as MG
    return MG.build_tiny(kind)[0].parameters()


@pytest.mark.parametrize("kind", ["marigold", "geowizard"])
def test_e2e_unet_gradients_with_checkpointing(kind):
    plain, plain2, ck = (_e2e_grads(kind, c) for c in (False, False, True))
    assert len(ck) == sum(1 for _ in _e2e_unet_params(kind))
    _equal_or_within_rerun_spread(plain, plain2, ck, f"{kind} UNet gradients")


# ------------------------------------------------------------------------------------------------ memory and reach
def _need_free(nbytes, what):
    torch.cuda.empty_cache()
    free, total = torch.cuda.mem_get_info()
    if free < nbytes:
        pytest.skip(f"{what} needs {nbytes / GB:.0f} GB free; the device has {free / GB:.1f} of {total / GB:.1f} GB free")


def _e2e_setup(res, batch):
    """SD-2-wide UNet (checkpointed, as in the recipes and bench.py's training leg) and VAE with seeded weights, and a
    batch whose depth target the engine's estimate explains (an affine map of it plus noise), as a real target does.
    A target independent of the estimate has a least-squares scale near 0 (1e-3 at 2048 x 2048): its SSI gradient
    then lies below fp16's subnormal range once the decoder's backward casts it, and the step has no gradient at all
    (DESIGN.md §8.6)."""
    from diffusion_e2e_ft_b200 import B200UNet2DConditionModel, DDIMScheduler
    from diffusion_e2e_ft_b200.training import e2e_ft_forward
    torch.manual_seed(4321)
    with torch.device(DEV):
        unet = B200UNet2DConditionModel()
    unet.train().requires_grad_(True)
    unet.enable_gradient_checkpointing()
    vae = _full_vae()
    if res > 1536:
        vae.enable_xformers_memory_efficient_attention()
    g = torch.Generator(device=DEV).manual_seed(5)
    rgb = torch.rand(batch, 3, res, res, device=DEV, generator=g) * 2 - 1
    mask = torch.ones(batch, 1, res, res, device=DEV, dtype=torch.bool)
    ctx = torch.randn(1, 77, 1024, device=DEV, generator=g) * 0.5
    _, est = e2e_ft_forward(unet, vae, DDIMScheduler(), rgb, torch.ones_like(mask, dtype=torch.float32), mask, ctx)
    depth = (5.0 + 3.0 * est + 0.3 * torch.randn(est.shape, device=DEV, generator=g)).clamp(0.1, 10.0)
    del est
    return unet, vae, DDIMScheduler(), (rgb, depth, mask, ctx)


def _e2e_step(unet, vae, sched, data):
    """One micro-step; returns its peak allocated memory and the share of UNet gradient entries that are nonzero."""
    from diffusion_e2e_ft_b200.training import LOSS_SCALE, e2e_ft_loss
    unet.zero_grad(set_to_none=True)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    loss, _ = e2e_ft_loss(unet, vae, sched, *data, "depth")
    (loss * LOSS_SCALE).backward()
    torch.cuda.synchronize()
    grads = [p.grad for p in unet.parameters()]
    assert all(g is not None and torch.isfinite(g).all() for g in grads)
    nonzero = sum(int(g.count_nonzero()) for g in grads) / sum(g.numel() for g in grads)
    print(f"loss {loss.item():.4g}, nonzero share of the UNet gradient entries {nonzero:.4f}")
    return torch.cuda.max_memory_allocated(), nonzero


def test_checkpointing_lowers_the_peak_at_768_bs2():
    """The recipe's shape (--train_batch_size 2, 768 x 768), UNet checkpointing on as in bench.py's training leg."""
    _need_free(32 * GB, "a 768^2 bs 2 micro-step without decoder checkpointing (23.0 GiB measured)")
    unet, vae, sched, data = _e2e_setup(768, 2)
    peaks = {}
    for ckpt in (False, True, False, True):
        (vae.enable_gradient_checkpointing if ckpt else vae.disable_gradient_checkpointing)()
        peaks[ckpt], nonzero = _e2e_step(unet, vae, sched, data)
        assert nonzero > 0.9
    print(f"E2E micro-step 768^2 bs 2 peak allocated: decoder checkpointing off {peaks[False] / GB:.2f} GiB, "
          f"on {peaks[True] / GB:.2f} GiB")
    assert peaks[True] < peaks[False], peaks


def test_e2e_step_at_2048_with_checkpointing():
    """2048 x 2048 bs 1 with both checkpointings and the memory-efficient attention: it fits, and it trains: its
    gradients are finite and nearly all UNet gradient entries are nonzero."""
    _need_free(56 * GB, "a 2048^2 micro-step (47.8 GiB measured)")
    unet, vae, sched, data = _e2e_setup(2048, 1)
    vae.enable_gradient_checkpointing()
    peak, nonzero = _e2e_step(unet, vae, sched, data)
    print(f"E2E micro-step 2048^2 bs 1 peak allocated {peak / GB:.2f} GiB")
    assert nonzero > 0.9
