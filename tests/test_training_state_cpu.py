"""Parameter groups, LR schedules and save / resume of the training state on the CPU, with the kernels replaced by
their plain-torch contracts (tests/cpu_emulation.py plus the ABI-11 grouped AdamW below): against torch.optim.AdamW
with the reference's groups + clip_grad_norm_, torch's LambdaLR stepped as accelerate steps it, the reference's own
IterExponential values (tests/golden/lr_schedule_pins.json), and torch's optimizer / scheduler state_dict layouts."""
import json
import math
import os
import random

import numpy as np
import pytest
import torch

import cpu_emulation
import engine_checks as EC           # also puts tests/golden on sys.path
from diffusion_e2e_ft_b200 import ops, training

HERE = os.path.dirname(os.path.abspath(__file__))


# ---- plain-torch contract of b200_adamw_step_state_groups (include/b200_e2eft.h, ABI 11)
def adamw_step_state_groups(param, grad, exp_avg, exp_avg_sq, state, grad_norm_sq_t, run_start, run_group, group_lr,
                            group_wd, betas=(0.9, 0.999), eps=1e-8, max_grad_norm=0.0, inv_world=1.0, dynamic_scale=True,
                            growth_interval=2000, min_scale=1.0, max_scale=65536.0):
    nsq = float(grad_norm_sq_t)
    S = float(state[0])
    if not math.isfinite(nsq) or nsq == 0.0:
        state[3] += 1
        state[4] = 1
        if not math.isfinite(nsq) and dynamic_scale:
            state[0] = max(S * 0.5, min_scale)
            state[1] = 0
        return
    state[2] += 1
    state[4] = 0
    bounds = run_start.tolist() + [param.numel()]
    for r, k in enumerate(run_group.tolist()):
        sl = slice(bounds[r], bounds[r + 1])
        cpu_emulation.adamw_step(param[sl], grad[sl], exp_avg[sl], exp_avg_sq[sl], int(state[2]), group_lr[k], betas,
                                 eps, group_wd[k], grad_norm_sq_t, max_grad_norm, inv_world / S)
    if dynamic_scale:
        state[1] += 1
        if float(state[1]) >= growth_interval:
            state[0] = min(S * 2.0, max_scale)
            state[1] = 0


@pytest.fixture
def emulated(monkeypatch):
    cpu_emulation.install(monkeypatch)
    monkeypatch.setattr(ops, "adamw_step_state_groups", adamw_step_state_groups)
    monkeypatch.setattr(ops, "ema_update", lambda ema, p, omd: ema.sub_(float(omd) * (ema - p)))
    monkeypatch.setattr(ops, "FUSE_GN_STATS", False)


def _unet(kind="geowizard"):
    import make_golden as MG
    ref, _ = MG.build_tiny(kind)
    unet, _ = EC.engine_from_oracle(ref, None, "cpu")
    unet.requires_grad_(True)
    return unet


def _grads(tr, seed, scale=1e-2):
    """Per-parameter gradients {name: tensor} and their flat layout."""
    g = torch.Generator().manual_seed(seed)
    per = {name: torch.randn(shape, generator=g) * scale for name, _, shape in tr._layout}
    flat = torch.zeros_like(tr.flat_param)
    for name, off, shape in tr._layout:
        flat[off:off + math.prod(shape)] = per[name].reshape(-1)
    return per, flat


def _rel(a, b):
    return float((a - b).norm() / b.norm())


def _step_with(tr, flat):
    tr.flat_grad.copy_(flat * tr.loss_scale())
    tr._micro, tr._synced = 0, True
    tr.step()


def _torch_groups(unet, groups, lr, params=None):
    """The reference's AdamW groups over `params` (name -> tensor), built as train.py:346-353 (one group) or
    train_depth_normal.py:428-444 (two groups)."""
    named = [(n, params[n]) for n, _ in unet.named_parameters()]
    if groups == 1:
        return [dict(params=[p for _, p in named], lr=lr)]
    return [dict(params=[p for n, p in named if "class_embedding" not in n], lr=lr),
            dict(params=[p for n, p in named if "class_embedding" in n], lr=lr * 10.0)]


# ---- parameter groups
def test_geowizard_groups_and_run_table():
    unet = _unet()
    tr = training.FlatTrainer(unet, lr=1e-3, param_groups=training.geowizard_param_groups())
    names = [n for n, _ in unet.named_parameters()]
    ce = [n for n in names if "class_embedding" in n]
    assert ce and tr._group_def[1]["params"] == ce and tr._group_def[1]["lr_mult"] == 10.0
    assert tr._group_def[0]["params"] == [n for n in names if "class_embedding" not in n]
    assert [r[1] for r in tr._runs] == [0, 1, 0] and all(r[0] % 4 == 0 for r in tr._runs)
    # the runs cover exactly the class-embedding views
    lo, hi = tr._runs[1][0], tr._runs[2][0]
    inside = {n for n, off, _ in tr._layout if lo <= off < hi}
    assert inside == set(ce)
    with pytest.raises(ValueError, match="no parameter group"):
        training.FlatTrainer(_unet(), param_groups=[dict(select=lambda n: "class_embedding" in n)])


def test_grouped_adamw_matches_torch_two_groups_with_clip_and_skips(emulated):
    """5 steps against torch.optim.AdamW with GeoWizard's two groups + clip_grad_norm_: a zero gradient (skipped:
    nothing moves, scale kept) and a non-finite one (skipped, scale halves) in between."""
    unet = _unet()
    tr = training.FlatTrainer(unet, lr=1e-3, max_grad_norm=1.0, param_groups=training.geowizard_param_groups(10))
    ref = {n: torch.nn.Parameter(p.detach().clone()) for n, p in unet.named_parameters()}
    opt = torch.optim.AdamW(_torch_groups(unet, 2, 1e-3, ref), lr=1e-3, betas=(0.9, 0.999), weight_decay=1e-2, eps=1e-8)
    for k in range(5):
        per, flat = _grads(tr, 30 + k, scale=(3.0 if k == 1 else 1e-2))
        keep = [t.clone() for t in (tr.flat_param, tr.exp_avg, tr.exp_avg_sq)]
        scale = tr.loss_scale()
        if k == 2:
            flat.zero_()
        if k == 3:
            flat[11] = float("inf")
        _step_with(tr, flat)
        if k in (2, 3):
            assert all(torch.equal(a, b) for a, b in zip(keep, (tr.flat_param, tr.exp_avg, tr.exp_avg_sq)))
            assert tr.loss_scale() == (scale if k == 2 else scale / 2)
            continue
        for n, p in ref.items():
            p.grad = per[n].clone()
        torch.nn.utils.clip_grad_norm_(list(ref.values()), 1.0)
        opt.step()
        for n, p in unet.named_parameters():
            assert _rel(p.detach(), ref[n].detach()) <= 2e-6, (k, n)   # kernel_checks.check_adamw_state's gate
            st = opt.state[ref[n]]
            off = dict((nm, o) for nm, o, _ in tr._layout)[n]
            m_ref = st["exp_avg"].reshape(-1)                  # the clip coefficients differ in the last bits
            assert (tr.exp_avg[off:off + p.numel()] - m_ref).norm() <= 1e-5 * m_ref.norm(), (k, n)
    assert tr.applied_steps() == 3 and tr.skipped_steps() == 2


# ---- LR schedules
def test_iter_exponential_matches_reference_pins():
    pins = json.load(open(os.path.join(HERE, "golden", "lr_schedule_pins.json")))
    for p in pins:
        f = training.IterExponential(p["total_iter_length"], p["final_ratio"], p["warmup_steps"])
        assert vars(f) == p["attributes"]
        assert [float(f(i)) for i in p["n_iter"]] == p["value"], p["total_iter_length"]
    assert training.ConstantLR(100)(0) == 1.0 and training.ConstantLR()(12345) == 1.0


class _Toy(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.conv_in = torch.nn.Linear(3, 5)
        self.class_embedding = torch.nn.Linear(2, 7)
        self.conv_out = torch.nn.Linear(5, 2)


@pytest.mark.filterwarnings("ignore:Detected call of")          # the dummy optimizer never steps
@pytest.mark.parametrize("N", [1, 2])
def test_applied_learning_rates_match_lambdalr_under_accelerate(emulated, monkeypatch, N):
    """250 optimizer steps: the rates handed to the kernel equal torch's LambdaLR(IterExponential(20000 N, 0.01,
    100 N)) stepped N times per optimizer step (accelerate's scheduler wrapper), lr = 0 on step 0 included."""
    seen = []
    monkeypatch.setattr(ops, "adamw_step_state_groups", lambda *a, **k: (seen.append(list(a[8])), adamw_step_state_groups(*a, **k)))
    torch.manual_seed(0)
    toy = _Toy()
    sched_fn = training.IterExponential(20000 * N, 0.01, 100 * N)
    tr = training.FlatTrainer(toy, lr=3e-5, param_groups=training.geowizard_param_groups(10), lr_schedule=sched_fn,
                              num_processes=N)
    opt = torch.optim.AdamW([dict(params=[torch.zeros(1, requires_grad=True)], lr=3e-5),
                             dict(params=[torch.zeros(1, requires_grad=True)], lr=3e-5 * 10.0)])
    ref = torch.optim.lr_scheduler.LambdaLR(opt, sched_fn)
    for k in range(250):
        assert tr.get_last_lr() == ref.get_last_lr(), k
        tr.flat_grad.fill_(0.0 if k % 7 == 3 else 1.0)             # device-skipped steps advance the schedule too
        tr._micro, tr._synced = 0, True
        tr.step()
        assert seen[-1] == [g["lr"] for g in opt.param_groups], k
        for _ in range(N):
            ref.step()
    assert seen[0] == [0.0, 0.0] and seen[100][0] > 0
    assert tr.skipped_steps() == len([k for k in range(250) if k % 7 == 3])
    with pytest.raises(ValueError, match="exclusive"):
        tr.step(lr=1e-4)
    with pytest.raises(ValueError, match="exclusive"):
        tr.micro_step(torch.zeros(()), lr=1e-4)


def test_without_schedule_lr_override_keeps_working(emulated, monkeypatch):
    seen = []
    monkeypatch.setattr(ops, "adamw_step_state_groups", lambda *a, **k: (seen.append(list(a[8])), adamw_step_state_groups(*a, **k)))
    tr = training.FlatTrainer(_Toy(), lr=2e-5, param_groups=training.geowizard_param_groups(10))
    assert tr.get_last_lr() == [2e-5, 2e-5 * 10.0]
    tr.flat_grad.fill_(1.0)
    tr.step(lr=1e-3)
    assert seen == [[1e-3, 1e-3 * 10.0]]


# ---- save / resume
def _loop_step(unet, tr, draws):
    x = torch.randn(2, 8, 16, 16)                                  # the global RNG, as the recipes draw their noise
    draws.append(x)
    c = torch.linspace(-1, 1, 2 * 96).reshape(2, 1, 96) * 0.5
    cl = torch.linspace(-0.5, 0.5, 20).reshape(2, 10)
    y = unet(x, 999, c, class_labels=cl).sample
    assert tr.micro_step((y * y).mean())


def _trainer(unet, **kw):
    kw.setdefault("param_groups", training.geowizard_param_groups(10))
    return training.FlatTrainer(unet, lr=1e-3, use_ema=True, lr_schedule=training.IterExponential(10, 0.1, 2), **kw)


def _snapshot(tr):
    return [t.clone() for t in (tr.flat_param, tr.exp_avg, tr.exp_avg_sq, tr.state, tr.ema)]


def test_resume_continues_bit_identically(emulated, tmp_path):
    torch.manual_seed(5)
    unet = _unet()
    tr = _trainer(unet)
    straight = []
    for _ in range(4):
        _loop_step(unet, tr, straight)
    want = _snapshot(tr)

    torch.manual_seed(5)
    unet = _unet()
    tr = _trainer(unet)
    split = []
    for _ in range(2):
        _loop_step(unet, tr, split)
    tr.save_state(str(tmp_path / "checkpoint-2"))
    torch.manual_seed(999)                                          # the resumed process starts with other RNG states
    unet2 = _unet()
    tr2 = _trainer(unet2)
    assert tr2.load_state(str(tmp_path / "checkpoint-2")) == 2
    assert tr2.step_count == 2 and tr2.ema_steps == 2 and tr2.get_last_lr() == tr.get_last_lr()
    for _ in range(2):
        _loop_step(unet2, tr2, split)
    assert all(torch.equal(a, b) for a, b in zip(straight, split))
    got = _snapshot(tr2)
    for name, a, b in zip(("param", "exp_avg", "exp_avg_sq", "state", "ema"), want, got):
        assert torch.equal(a, b), name


def test_rng_states_round_trip(emulated, tmp_path):
    tr = training.FlatTrainer(_unet("marigold"))
    random.seed(1), np.random.seed(2), torch.manual_seed(3)
    tr.save_state(str(tmp_path))
    want = (random.random(), np.random.rand(), torch.rand(3))
    random.seed(7), np.random.seed(8), torch.manual_seed(9)
    tr.load_state(str(tmp_path))
    got = (random.random(), np.random.rand(), torch.rand(3))
    assert want[0] == got[0] and want[1] == got[1] and torch.equal(want[2], got[2])


@pytest.mark.parametrize("groups", [1, 2])
def test_optimizer_and_scheduler_files_load_into_torch(emulated, tmp_path, groups):
    """optimizer.bin / scheduler.bin load into torch's AdamW / LambdaLR built as the reference builds them; one more
    step of each from there agrees."""
    kind = "geowizard" if groups == 2 else "marigold"
    unet = _unet(kind)
    pg = training.geowizard_param_groups(10) if groups == 2 else None
    sched_fn = training.IterExponential(20, 0.01, 3)
    tr = training.FlatTrainer(unet, lr=1e-3, max_grad_norm=1.0, param_groups=pg, lr_schedule=sched_fn, num_processes=2)
    for k in range(5):
        _step_with(tr, _grads(tr, 50 + k)[1])
    tr.save_state(str(tmp_path))
    ref = {n: torch.nn.Parameter(p.detach().clone()) for n, p in unet.named_parameters()}
    opt = torch.optim.AdamW(_torch_groups(unet, groups, 1e-3, ref), lr=1e-3, betas=(0.9, 0.999), weight_decay=1e-2,
                            eps=1e-8)
    sched = torch.optim.lr_scheduler.LambdaLR(opt, training.IterExponential(20, 0.01, 3))
    opt.load_state_dict(torch.load(tmp_path / "optimizer.bin"))
    sched.load_state_dict(torch.load(tmp_path / "scheduler.bin"))
    assert sched.get_last_lr() == tr.get_last_lr() and sched.last_epoch == 10
    assert vars(sched.lr_lambdas[0]) == vars(sched_fn)
    assert all(float(s["step"]) == 5.0 for s in opt.state.values()) and len(opt.state) == len(ref)
    per, flat = _grads(tr, 60)
    for n, p in ref.items():
        p.grad = per[n].clone()
    torch.nn.utils.clip_grad_norm_(list(ref.values()), 1.0)
    opt.step()
    _step_with(tr, flat)
    for n, p in unet.named_parameters():
        assert _rel(p.detach(), ref[n].detach()) <= 1e-6, n


def test_reference_style_folder_without_engine_state_loads(emulated, tmp_path):
    """A folder as the reference writes it: unet/, optimizer.bin from torch's AdamW, scheduler.bin from LambdaLR,
    no flat_trainer.pt.  Loads with the default loss scale and applied steps = the optimizer's step."""
    unet = _unet()
    ref = {n: torch.nn.Parameter(p.detach().clone()) for n, p in unet.named_parameters()}
    opt = torch.optim.AdamW(_torch_groups(unet, 2, 1e-3, ref), lr=1e-3, weight_decay=1e-2)
    sched = torch.optim.lr_scheduler.LambdaLR(opt, training.IterExponential(40, 0.01, 4))
    g = torch.Generator().manual_seed(3)
    for _ in range(3):
        for p in ref.values():
            p.grad = torch.randn(p.shape, generator=g) * 1e-2
        opt.step()
        sched.step()
    unet.save_pretrained(str(tmp_path / "unet"), state_dict={n: p.detach() for n, p in ref.items()})
    torch.save(opt.state_dict(), tmp_path / "optimizer.bin")
    torch.save(sched.state_dict(), tmp_path / "scheduler.bin")
    tr = training.FlatTrainer(_unet(), lr=1e-3, param_groups=training.geowizard_param_groups(10),
                              lr_schedule=training.IterExponential(40, 0.01, 4), loss_scale=256.0)
    assert tr.load_state(str(tmp_path)) == 3
    assert tr.loss_scale() == 256.0 and tr.applied_steps() == 3 and tr.skipped_steps() == 0
    assert tr.get_last_lr() == sched.get_last_lr()
    for n, p in tr.module.named_parameters():
        assert torch.equal(p.detach(), ref[n].detach()), n
        off = dict((nm, o) for nm, o, _ in tr._layout)[n]
        assert torch.equal(tr.exp_avg_sq[off:off + p.numel()], opt.state[ref[n]]["exp_avg_sq"].reshape(-1))


def _saved(tmp_path, **kw):
    unet = _unet()
    tr = _trainer(unet, **kw)
    for k in range(2):
        _step_with(tr, _grads(tr, 70 + k)[1])
    tr.save_state(str(tmp_path))
    return tr


def _fresh_snapshot(**kw):
    tr = _trainer(_unet(), **kw)
    return tr, _snapshot(tr) + [torch.tensor([tr.step_count, tr.ema_steps])]


def _unchanged(tr, snap):
    now = _snapshot(tr) + [torch.tensor([tr.step_count, tr.ema_steps])]
    return all(torch.equal(a, b) for a, b in zip(snap, now))


def test_malformed_folders_raise_before_any_buffer_changes(emulated, tmp_path):
    from safetensors.torch import load_file, save_file
    _saved(tmp_path)
    # a group definition that differs from the trainer's
    tr, snap = _fresh_snapshot(param_groups=training.geowizard_param_groups(5))
    with pytest.raises(ValueError, match="parameter groups"):
        tr.load_state(str(tmp_path))
    assert _unchanged(tr, snap)
    # ... also without flat_trainer.pt (sizes from optimizer.bin)
    os.rename(tmp_path / "flat_trainer.pt", tmp_path / "ft.bak")
    tr, snap = _fresh_snapshot(param_groups=None)
    with pytest.raises(ValueError, match="parameter groups"):
        tr.load_state(str(tmp_path))
    assert _unchanged(tr, snap)
    os.rename(tmp_path / "ft.bak", tmp_path / "flat_trainer.pt")
    # per-parameter steps that differ
    opt = torch.load(tmp_path / "optimizer.bin")
    good = {k: dict(v) for k, v in opt["state"].items()}
    opt["state"][3]["step"] = torch.tensor(1.0)
    torch.save(opt, tmp_path / "optimizer.bin")
    tr, snap = _fresh_snapshot()
    with pytest.raises(ValueError, match="steps"):
        tr.load_state(str(tmp_path))
    assert _unchanged(tr, snap)
    opt["state"] = good
    torch.save(opt, tmp_path / "optimizer.bin")
    # a parameter of the wrong shape, then a missing one
    path = tmp_path / "unet" / "diffusion_pytorch_model.safetensors"
    sd = {k: v.clone() for k, v in load_file(str(path)).items()}      # not the memory map of the file rewritten below
    name = next(n for n in sd if n.endswith("conv_in.weight"))
    bad = dict(sd)
    bad[name] = sd[name][:, :4].contiguous()
    save_file(bad, str(path))
    tr, snap = _fresh_snapshot()
    with pytest.raises(ValueError, match="conv_in.weight"):
        tr.load_state(str(tmp_path))
    assert _unchanged(tr, snap)
    del bad[name]
    save_file(bad, str(path))
    with pytest.raises(ValueError, match="conv_in.weight"):
        tr.load_state(str(tmp_path))
    assert _unchanged(tr, snap)
    save_file(sd, str(path))
    assert tr.load_state(str(tmp_path)) == 2 and not _unchanged(tr, snap)


def test_save_state_only_at_window_boundary(emulated, tmp_path):
    tr = training.FlatTrainer(_Toy(), accumulation_steps=2)
    tr.backward(tr.module.conv_out(tr.module.conv_in(torch.ones(1, 3))).sum())
    with pytest.raises(RuntimeError, match="accumulation window"):
        tr.save_state(str(tmp_path))
    assert not os.listdir(tmp_path)


def test_latest_checkpoint_and_pruning(tmp_path):
    assert training.latest_checkpoint(str(tmp_path / "missing")) is None
    assert training.latest_checkpoint(str(tmp_path)) is None
    for d in ("checkpoint-900", "checkpoint-1000", "checkpoint-50", "logs", "checkpoint-7"):
        os.makedirs(tmp_path / d)
    assert training.latest_checkpoint(str(tmp_path)) == str(tmp_path / "checkpoint-1000")      # numeric, not lexical
    assert training.prune_checkpoints(str(tmp_path), None) == []
    assert training.prune_checkpoints(str(tmp_path), 5) == []                                  # 4 < 5: room for one
    removed = training.prune_checkpoints(str(tmp_path), 3)                                       # keep limit - 1 = 2
    assert removed == [str(tmp_path / "checkpoint-7"), str(tmp_path / "checkpoint-50")]
    assert sorted(os.listdir(tmp_path)) == ["checkpoint-1000", "checkpoint-900", "logs"]


def test_two_rank_gloo_save_and_resume(tmp_path):
    """world_size 2 on gloo, kernels emulated: only rank 0 writes the shared files, every rank its own RNG file; both
    ranks resume to identical parameters and each gets its own RNG state back."""
    import subprocess
    import sys
    root = os.path.dirname(HERE)
    code = r'''
import os, sys, torch, torch.distributed as dist
torch.set_num_threads(2)
sys.path.insert(0, %r); sys.path.insert(0, %r + "/tests"); sys.path.insert(0, %r + "/tests/golden")
import cpu_emulation, engine_checks as E, make_golden as MG, test_training_state_cpu as T
from diffusion_e2e_ft_b200 import ops, training
class MP:
    def setattr(self, o, n, v): setattr(o, n, v)
cpu_emulation.install(MP()); ops.FUSE_GN_STATS = False
ops.adamw_step_state_groups = T.adamw_step_state_groups
ops.ema_update = lambda ema, p, omd: ema.sub_(float(omd) * (ema - p))
r = int(sys.argv[1]); out = sys.argv[2]
dist.init_process_group("gloo", init_method="tcp://127.0.0.1:29593", rank=r, world_size=2)
torch.manual_seed(100 + r)
unet = T._unet()
tr = T._trainer(unet)
draws = []
T._loop_step(unet, tr, draws)
written = []
save, pretrained = torch.save, type(unet).save_pretrained
torch.save = lambda obj, f, *a, **k: (written.append(os.path.basename(str(f))), save(obj, f, *a, **k))[1]
type(unet).save_pretrained = lambda self, d, *a, **k: (written.append(os.path.basename(d)), pretrained(self, d, *a, **k))[1]
tr.save_state(out)
torch.save, type(unet).save_pretrained = save, pretrained
want_files = ["unet", "unet_ema", "optimizer.bin", "scheduler.bin", "flat_trainer.pt", "random_states_0.pkl"]
assert sorted(written) == sorted(want_files if r == 0 else ["random_states_1.pkl"]), written
saved = tr.flat_param.clone()
after = torch.randn(5)
T._loop_step(unet, tr, draws)
unet2 = T._unet(); tr2 = T._trainer(unet2)
assert tr2.load_state(out) == 1
assert torch.equal(tr2.flat_param, saved)
assert torch.equal(torch.randn(5), after), "RNG state of this rank"
both = [torch.zeros_like(saved) for _ in range(2)]
dist.all_gather(both, tr2.flat_param)
assert torch.equal(both[0], both[1])
rs = [torch.zeros(5) for _ in range(2)]
dist.all_gather(rs, after)
assert not torch.equal(rs[0], rs[1])
print("OK")
''' % (root, root, root)
    ps = [subprocess.Popen([sys.executable, "-c", code, str(r), str(tmp_path / "checkpoint-1")], stdout=subprocess.PIPE,
                           stderr=subprocess.PIPE, text=True) for r in range(2)]
    outs = [p.communicate(timeout=600) for p in ps]
    assert all(p.returncode == 0 for p in ps), outs
    assert all(o[0].strip().endswith("OK") for o in outs), outs
    assert sorted(os.listdir(tmp_path / "checkpoint-1")) == sorted(
        ["unet", "unet_ema", "optimizer.bin", "scheduler.bin", "flat_trainer.pt", "random_states_0.pkl",
         "random_states_1.pkl"])
