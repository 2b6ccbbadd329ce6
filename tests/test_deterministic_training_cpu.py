"""Source guard for bitwise-reproducible training (DESIGN.md §9 "Reduction order"): no floating-point atomic on the
training path's reductions, and their grids never depend on the device's SM count."""
import os
import re

import pytest

CSRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "diffusion_e2e_ft_b200", "csrc")
FLOAT_ATOMIC = re.compile(r"\batomic(Add|Sub)\s*\(|\bred\.[\w.:]*\.f(16|32|64)\b|\batom\.[\w.:]*\.f(16|32|64)\b")


def _src(name):
    with open(os.path.join(CSRC, name)) as f:
        return re.sub(r"//[^\n]*", "", f.read())     # comments may name what the code no longer does


def _function(src, name):
    """The text of the function `name` (through its matching closing brace)."""
    i = src.index(name)
    j = src.index("{", i)
    depth = 0
    for k in range(j, len(src)):
        depth += {"{": 1, "}": -1}.get(src[k], 0)
        if depth == 0:
            return src[i:k + 1]
    raise AssertionError(name)


@pytest.mark.parametrize("name", ["backward.cu", "loss.cu", "optim.cu"])
def test_no_atomics_in_training_reductions(name):
    # the integer atomics these files might use would be fine; none of their sums may be atomic
    hits = [m.group(0) for m in FLOAT_ATOMIC.finditer(_src(name))]
    assert not hits, (name, hits)


def test_no_atomics_in_gn_stats_kernel():
    body = _function(_src("norm.cu"), "__global__ void gn_stats_kernel")
    assert "cluster_add_partials" in body
    assert not FLOAT_ATOMIC.search(body)


def test_guard_sees_an_atomic():
    assert FLOAT_ATOMIC.search("atomicAdd(&s[0], v);") and FLOAT_ATOMIC.search('asm("red.global.add.f32 [%0], %1;")')
    assert not FLOAT_ATOMIC.search("cluster_add_partials(part, 1, f);")


@pytest.mark.parametrize("entry", ["b200_sumsq", "b200_col_sum", "b200_group_norm_bwd_sums", "b200_layer_norm_bwd",
                                   "b200_ssi_loss", "b200_angular_loss", "b200_masked_latent_mse",
                                   "b200_ssi_loss_bwd", "b200_angular_loss_bwd", "b200_group_norm_stats"])
def test_reduction_grids_do_not_read_the_sm_count(entry):
    for name in ("backward.cu", "loss.cu", "optim.cu", "norm.cu"):
        src = _src(name)
        if f'extern "C" int {entry}(' in src:
            body = _function(src, f'extern "C" int {entry}(')
            assert "sm_count" not in body and "launch_clustered" in body, (entry, name)
            return
    raise AssertionError(f"{entry} not found")
