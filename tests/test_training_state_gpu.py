"""The grouped fused AdamW kernel (ABI 11), GeoWizard's two parameter groups with the exponential LR schedule against
the oracle with torch.optim.AdamW + LambdaLR + clip_grad_norm_, and save / resume of the training state on the GPU."""
import pytest
import torch

import engine_checks as EC
import make_golden as MG
from diffusion_e2e_ft_b200 import DDIMScheduler, ops, training
from kernel_checks import _rand, rel_l2
from oracle import pipeline as OP

DEV = "cuda:0"
RUNS = ([0, 40000, 70000], [0, 1, 0])          # three runs: group 0, group 1, group 0 again
LRS, WDS = [3e-3, 3e-2], [1e-2, 0.0]


def _segments(x):
    return x[:40000], x[40000:70000], x[70000:]


@pytest.mark.gpu
def test_grouped_adamw_kernel_matches_torch_adamw_groups():
    """n = 100003, a 3-run table over 2 groups (own lr and weight decay) vs torch.optim.AdamW with the same groups +
    clip_grad_norm_: good steps with a loss-scaled, world-summed gradient, a non-finite gradient (skipped, scale
    halved), an all-zero one (skipped, scale kept), then scale growth — kernel_checks.check_adamw_state's sequence."""
    n, world = 100003, 4
    p0 = _rand(n, seed=71, dtype=torch.float32)
    refs = [torch.nn.Parameter(s.clone()) for s in _segments(p0)]
    opt = torch.optim.AdamW([dict(params=[refs[0], refs[2]], lr=LRS[0], weight_decay=WDS[0]),
                             dict(params=[refs[1]], lr=LRS[1], weight_decay=WDS[1])], betas=(0.9, 0.999), eps=1e-8)
    p = p0.clone()
    m, v = torch.zeros_like(p), torch.zeros_like(p)
    state = torch.zeros(8, dtype=torch.float32, device=DEV)
    state[0] = 1024.0
    table = ops.adamw_run_table(*RUNS, n, 2, DEV)
    worst = 0.0

    def engine_step(g_true):
        g = g_true * (float(state[0]) * world)
        ops.adamw_step_state_groups(p, g, m, v, state, ops.grad_norm_sq(g), *table, LRS, WDS, max_grad_norm=1.0,
                                    inv_world=1.0 / world, dynamic_scale=True, growth_interval=3)
        torch.cuda.synchronize()

    def ref_step(g_true):
        for r, s in zip(refs, _segments(g_true)):
            r.grad = s.clone()
        torch.nn.utils.clip_grad_norm_(refs, 1.0)
        opt.step()

    def err():
        return rel_l2(p, torch.cat([r.data for r in refs]))

    for step in range(1, 3):
        g = _rand(n, seed=71 + step, dtype=torch.float32) * (3.0 if step == 2 else 0.001)
        ref_step(g); engine_step(g)
        worst = max(worst, err())
    assert state.tolist()[:5] == [1024.0, 2.0, 2.0, 0.0, 0.0], state.tolist()
    keep = (p.clone(), m.clone(), v.clone())
    bad = _rand(n, seed=80, dtype=torch.float32)
    bad[5] = float("inf")
    engine_step(bad)
    assert all(torch.equal(a, b) for a, b in zip(keep, (p, m, v))) and state.tolist()[:5] == [512.0, 0.0, 2.0, 1.0, 1.0]
    engine_step(torch.zeros(n, device=DEV))
    assert all(torch.equal(a, b) for a, b in zip(keep, (p, m, v))) and state.tolist()[:5] == [512.0, 0.0, 2.0, 2.0, 1.0]
    for step in range(3, 6):
        g = _rand(n, seed=71 + step, dtype=torch.float32) * 0.01
        ref_step(g); engine_step(g)
        worst = max(worst, err())
    assert state.tolist()[:5] == [1024.0, 0.0, 5.0, 2.0, 0.0], state.tolist()
    assert worst <= 2e-6, worst
    for seg, r in zip(_segments(p), refs):
        assert rel_l2(seg, r.data) <= 2e-6


@pytest.mark.gpu
def test_grouped_kernel_with_one_run_is_bit_identical_to_adamw_step_state():
    n = 100003
    bufs = []
    for grouped in (False, True):
        p = _rand(n, seed=90, dtype=torch.float32)
        m, v = torch.zeros_like(p), torch.zeros_like(p)
        state = torch.tensor([1024.0, 0, 0, 0, 0, 0, 0, 0], device=DEV)
        table = ops.adamw_run_table([0], [0], n, 1, DEV)
        for step in range(5):
            g = _rand(n, seed=91 + step, dtype=torch.float32) * (2048.0 if step != 2 else 0.0)
            nsq = ops.grad_norm_sq(g)
            if grouped:
                ops.adamw_step_state_groups(p, g, m, v, state, nsq, *table, [3e-3], [1e-2], max_grad_norm=1.0,
                                            growth_interval=2)
            else:
                ops.adamw_step_state(p, g, m, v, state, nsq, lr=3e-3, weight_decay=1e-2, max_grad_norm=1.0,
                                     growth_interval=2)
        torch.cuda.synchronize()
        bufs.append((p, m, v, state))
    assert all(torch.equal(a, b) for a, b in zip(*bufs))


@pytest.mark.gpu
def test_run_table_is_checked_before_launch():
    with pytest.raises(ValueError, match="multiples of 4"):
        ops.adamw_run_table([0, 6], [0, 1], 100, 2, DEV)
    with pytest.raises(ValueError, match="groups must lie"):
        ops.adamw_run_table([0, 8], [0, 2], 100, 2, DEV)
    with pytest.raises(ValueError, match="runs"):
        ops.adamw_run_table(list(range(0, 4 * 1025, 4)), [0] * 1025, 10 ** 6, 1, DEV)


# ---- GeoWizard's groups and schedule on the tiny training loop
def _geowizard_batch(g, B=2):
    return (torch.rand(B, 3, 64, 64, generator=g) * 2 - 1, torch.randn(B, 1, 96, generator=g) * 0.5,
            torch.rand(B, 1, 64, 64, generator=g) > 0.2, torch.rand(B, 1, 64, 64, generator=g) * 9.9 + 0.1,
            torch.nn.functional.normalize(torch.randn(B, 3, 64, 64, generator=g), dim=1))


def _oracle_loss(unet_ref, vae_ref, rgb, emb, mask, gt_d, gt_n):
    B = rgb.shape[0]
    with torch.no_grad():
        lat = OP.encode_rgb(vae_ref, rgb)
    x = torch.cat([lat.repeat(2, 1, 1, 1), torch.zeros_like(lat).repeat(2, 1, 1, 1)], 1)
    cls = OP.geowizard_class_embedding("indoor", rgb.dtype, B)
    v = unet_ref(x, torch.full((2 * B,), 999), encoder_hidden_states=emb.repeat(2, 1, 1), class_labels=cls).sample
    dec = OP.decode_latent(vae_ref, OP.DDIMOneStep().pred_original_sample(v, 999, torch.zeros_like(v)))
    est_d = dec[:B].mean(1, keepdim=True).clamp(-1, 1)
    est_n = (dec[B:] / (dec[B:].norm(dim=1, keepdim=True) + 1e-5)).clamp(-1, 1)
    return 0.5 * OP.ssi_loss(est_d, gt_d, mask) + OP.angular_loss(est_n, -gt_n, mask)


def _engine_loop(param_groups, steps=3, lr=1e-4, schedule=lambda: training.IterExponential(20, 0.01, 2)):
    unet_ref, vae_ref = MG.build_tiny("geowizard")
    unet, vae = EC.engine_from_oracle(unet_ref, vae_ref, DEV)
    unet.requires_grad_(True)
    start = {n: p.detach().float().cpu().clone() for n, p in unet.named_parameters()}
    tr = training.FlatTrainer(unet, lr=lr, weight_decay=1e-2, max_grad_norm=1.0, param_groups=param_groups,
                              lr_schedule=schedule(), num_processes=1)
    g = torch.Generator().manual_seed(33)
    losses = []
    for _ in range(steps):
        rgb, emb, mask, gt_d, gt_n = _geowizard_batch(g)
        loss, _, _ = training.e2e_ft_loss_geowizard(unet, vae, DDIMScheduler(), rgb.to(DEV), gt_d.to(DEV),
                                                    gt_n.to(DEV), mask.to(DEV), emb.to(DEV), "indoor")
        tr.micro_step(loss)
        losses.append(loss.item())
    upd = {n: p.detach().float().cpu() - start[n] for n, p in unet.named_parameters()}
    return losses, upd, start


@pytest.mark.gpu
def test_geowizard_groups_and_schedule_match_oracle_adamw():
    """train_depth_normal.py:428-481,640-791 for 3 optimizer steps: engine FlatTrainer with geowizard_param_groups(10)
    and IterExponential vs the oracle graph with torch AdamW (two groups) + LambdaLR + clip_grad_norm_.  Gates of
    test_training_loop_matches_oracle_adamw; the class-embedding update is ~10x the single-group one."""
    lr = 1e-4
    unet_ref, vae_ref = MG.build_tiny("geowizard")
    unet_ref.requires_grad_(True)
    vae_ref.requires_grad_(False)
    start = {n: p.detach().clone() for n, p in unet_ref.named_parameters()}
    params, params_ce = [], []
    for n, p in unet_ref.named_parameters():
        (params_ce if "class_embedding" in n else params).append(p)
    opt = torch.optim.AdamW([dict(params=params, lr=lr), dict(params=params_ce, lr=lr * 10.0)], betas=(0.9, 0.999),
                            weight_decay=1e-2, eps=1e-8)
    sched = torch.optim.lr_scheduler.LambdaLR(opt, training.IterExponential(20, 0.01, 2))
    g = torch.Generator().manual_seed(33)
    lo = []
    for _ in range(3):
        loss = _oracle_loss(unet_ref, vae_ref, *_geowizard_batch(g))
        opt.zero_grad()
        loss.backward()
        torch.nn.utils.clip_grad_norm_(unet_ref.parameters(), 1.0)
        opt.step()
        sched.step()
        lo.append(loss.item())
    le, upd, _ = _engine_loop(training.geowizard_param_groups(10), lr=lr)
    for a, b in zip(le, lo):
        assert abs(a - b) / abs(b) <= 3e-3, (le, lo)
    dot = ne = no = 0.0
    for n, p in unet_ref.named_parameters():
        do = p.detach() - start[n]
        dot += (upd[n] * do).sum().item()
        ne += upd[n].pow(2).sum().item()
        no += do.pow(2).sum().item()
    assert dot / (ne * no) ** 0.5 >= 0.98 and abs((ne / no) ** 0.5 - 1.0) <= 0.03, (dot / (ne * no) ** 0.5, (ne / no) ** 0.5)
    # against one group at the base rate: the class-embedding projection moves ~10x as far, the rest about as far
    _, upd1, _ = _engine_loop(None, lr=lr)

    def norm(u, ce):
        return sum(v.pow(2).sum().item() for n, v in u.items() if ("class_embedding" in n) == ce) ** 0.5
    ratio = norm(upd, True) / norm(upd1, True)
    assert 8.0 <= ratio <= 12.0, ratio
    assert 0.8 <= norm(upd, False) / norm(upd1, False) <= 1.25


# ---- save / resume
def _opt_trainer(max_grad_norm, use_ema=True):
    unet_ref, _ = MG.build_tiny("geowizard")
    unet, _ = EC.engine_from_oracle(unet_ref, None, DEV)
    unet.requires_grad_(True)
    return training.FlatTrainer(unet, lr=1e-3, max_grad_norm=max_grad_norm, use_ema=use_ema,
                                param_groups=training.geowizard_param_groups(10),
                                lr_schedule=training.IterExponential(10, 0.1, 2))


def _write_grads(tr, k):
    g = torch.Generator().manual_seed(200 + k)
    tr.flat_grad.copy_((torch.randn(tr.flat_grad.shape, generator=g) * 1e-2 * tr.loss_scale()).to(DEV))
    tr._micro, tr._synced = 0, True
    tr.step()


def _bufs(tr):
    return [t.detach().clone() for t in (tr.flat_param, tr.exp_avg, tr.exp_avg_sq, tr.state, tr.ema)]


@pytest.mark.gpu
@pytest.mark.parametrize("max_grad_norm,tol", [(0.0, 0.0), (1.0, 1e-6)])
def test_optimizer_resume(tmp_path, max_grad_norm, tol):
    """Gradients written into flat_grad: 4 steps straight vs 2 + save_state + a fresh trainer's load_state + 2.
    Bit-identical without clipping; with it, the norm's atomically ordered sum of squares leaves <= 1e-6."""
    tr = _opt_trainer(max_grad_norm)
    for k in range(4):
        _write_grads(tr, k)
    want = _bufs(tr)
    tr = _opt_trainer(max_grad_norm)
    for k in range(2):
        _write_grads(tr, k)
    tr.save_state(str(tmp_path / "checkpoint-2"))
    tr2 = _opt_trainer(max_grad_norm)
    assert tr2.load_state(training.latest_checkpoint(str(tmp_path))) == 2
    for k in range(2, 4):
        _write_grads(tr2, k)
    torch.cuda.synchronize()
    for name, a, b in zip(("param", "exp_avg", "exp_avg_sq", "state", "ema"), want, _bufs(tr2)):
        if tol == 0.0:
            assert torch.equal(a, b), name
        elif name == "state":                       # [5] is the clip coefficient itself; the rest is exact
            assert torch.equal(a[torch.arange(8) != 5], b[torch.arange(8) != 5]), (a, b)
        else:
            assert rel_l2(b, a) <= tol, (name, rel_l2(b, a))


@pytest.mark.gpu
def test_full_loop_resume(tmp_path):
    """The tiny GeoWizard loop (forward, loss-scaled backward, clip, grouped AdamW, EMA): 4 steps straight vs
    2 + save + load + 2.  GroupNorm-backward sums use global atomics, so two uninterrupted runs are not bit-identical
    either: <= 1e-5 relative on the parameters, or within twice the spread of two uninterrupted runs."""
    def loop(tr, unet, vae, g, steps):
        for _ in range(steps):
            rgb, emb, mask, gt_d, gt_n = _geowizard_batch(g)
            loss, _, _ = training.e2e_ft_loss_geowizard(unet, vae, DDIMScheduler(), rgb.to(DEV), gt_d.to(DEV),
                                                        gt_n.to(DEV), mask.to(DEV), emb.to(DEV), "indoor")
            tr.micro_step(loss)

    def build():
        unet_ref, vae_ref = MG.build_tiny("geowizard")
        unet, vae = EC.engine_from_oracle(unet_ref, vae_ref, DEV)
        unet.requires_grad_(True)
        tr = training.FlatTrainer(unet, lr=1e-4, use_ema=True, param_groups=training.geowizard_param_groups(10),
                                  lr_schedule=training.IterExponential(20, 0.01, 2))
        return tr, unet, vae

    straight = []
    for _ in range(2):                          # twice: the run-to-run spread of the atomically ordered sums
        tr, unet, vae = build()
        g = torch.Generator().manual_seed(41)
        loop(tr, unet, vae, g, 4)
        straight.append(_bufs(tr))
    tr, unet, vae = build()
    g = torch.Generator().manual_seed(41)
    loop(tr, unet, vae, g, 2)
    tr.save_state(str(tmp_path))
    tr2, unet2, vae2 = build()
    tr2.load_state(str(tmp_path))
    loop(tr2, unet2, vae2, g, 2)
    got = _bufs(tr2)
    assert tr2.step_count == 4 and tr2.applied_steps() == tr.applied_steps() + 2
    want, again = straight
    for name, i in (("param", 0), ("exp_avg", 1), ("ema", 4)):
        spread, err = rel_l2(again[i], want[i]), rel_l2(got[i], want[i])
        # Adam's normalised step turns last-bit gradient noise into up to +-lr on near-zero gradients, so two
        # uninterrupted runs differ too: the resumed run must be as close to the first as the second one is
        assert err <= max(1e-5, 2.0 * spread), (name, err, spread)
