"""ORACLE (test infrastructure) — fp32 PyTorch restatement of the CLIP TEXT encoder the Marigold pipeline calls once
per process for the empty prompt (Marigold/marigold/marigold_pipeline.py:355-369: tokenizer("", padding="do_not_pad")
-> `self.text_encoder(text_input_ids)[0]` -> `empty_text_embed` [1, 2, 1024]).

The implementation lives in a third-party dependency, transformers==4.37.2 (requirements.txt:7), absent from
the reference checkout: `models/clip/modeling_clip.py` — CLIPTextEmbeddings (token + learned position embedding),
CLIPEncoderLayer (pre-LN; causal multi-head self-attention with q scaled by head_dim**-0.5; MLP fc1 -> act -> fc2),
final_layer_norm, pooled output = the hidden state at the EOS position.  Restated here from that published
algorithm with the transformers `state_dict` names, and PINNED in tests/test_clip_text.py against the installed
transformers (5.5.0 here: same arithmetic) with shared random weights.  Only tests/ may import this module.
"""
from dataclasses import dataclass

import torch
import torch.nn.functional as F


@dataclass
class CLIPTextCfg:
    vocab_size: int = 49408
    hidden_size: int = 1024                 # stabilityai/stable-diffusion-2 text_encoder/config.json
    intermediate_size: int = 4096
    num_hidden_layers: int = 23
    num_attention_heads: int = 16
    max_position_embeddings: int = 77
    layer_norm_eps: float = 1e-5
    hidden_act: str = "gelu"
    eos_token_id: int = 49407
    bos_token_id: int = 49406


def tiny_clip_cfg(**kw):
    base = dict(hidden_size=128, intermediate_size=256, num_hidden_layers=2, num_attention_heads=2)
    base.update(kw)
    return CLIPTextCfg(**base)


def _act(x, name):
    if name == "gelu":
        return F.gelu(x)
    if name == "quick_gelu":
        return x * torch.sigmoid(1.702 * x)
    raise ValueError(name)


def random_state_dict(cfg: CLIPTextCfg, seed=0, dtype=torch.float32):
    """Seeded weights in the transformers layout (scaled so 23 layers stay O(1))."""
    g = torch.Generator().manual_seed(seed)
    C, I = cfg.hidden_size, cfg.intermediate_size
    sd = {}

    def rn(*shape, s=1.0):
        return (torch.randn(*shape, generator=g) * s).to(dtype)
    sd["text_model.embeddings.token_embedding.weight"] = rn(cfg.vocab_size, C, s=0.5)
    sd["text_model.embeddings.position_embedding.weight"] = rn(cfg.max_position_embeddings, C, s=0.5)
    for i in range(cfg.num_hidden_layers):
        p = f"text_model.encoder.layers.{i}."
        for n in ("q_proj", "k_proj", "v_proj", "out_proj"):
            sd[p + f"self_attn.{n}.weight"] = rn(C, C, s=C ** -0.5)
            sd[p + f"self_attn.{n}.bias"] = rn(C, s=0.1)
        for n in ("layer_norm1", "layer_norm2"):
            sd[p + n + ".weight"] = 1.0 + rn(C, s=0.1)
            sd[p + n + ".bias"] = rn(C, s=0.1)
        sd[p + "mlp.fc1.weight"] = rn(I, C, s=C ** -0.5)
        sd[p + "mlp.fc1.bias"] = rn(I, s=0.1)
        sd[p + "mlp.fc2.weight"] = rn(C, I, s=I ** -0.5)
        sd[p + "mlp.fc2.bias"] = rn(C, s=0.1)
    sd["text_model.final_layer_norm.weight"] = 1.0 + rn(C, s=0.1)
    sd["text_model.final_layer_norm.bias"] = rn(C, s=0.1)
    return sd


@torch.no_grad()
def clip_text_forward(sd, cfg: CLIPTextCfg, input_ids: torch.Tensor):
    """-> (last_hidden_state [B, L, C], pooler_output [B, C]) in fp32."""
    sd = {k: v.float() for k, v in sd.items()}
    B, L = input_ids.shape
    C, H = cfg.hidden_size, cfg.num_attention_heads
    d = C // H
    h = sd["text_model.embeddings.token_embedding.weight"][input_ids] \
        + sd["text_model.embeddings.position_embedding.weight"][:L][None]
    causal = torch.full((L, L), float("-inf")).triu(1)                       # key j > query i is hidden
    for i in range(cfg.num_hidden_layers):
        p = f"text_model.encoder.layers.{i}."
        y = F.layer_norm(h, (C,), sd[p + "layer_norm1.weight"], sd[p + "layer_norm1.bias"], cfg.layer_norm_eps)
        q = F.linear(y, sd[p + "self_attn.q_proj.weight"], sd[p + "self_attn.q_proj.bias"]) * d ** -0.5
        k = F.linear(y, sd[p + "self_attn.k_proj.weight"], sd[p + "self_attn.k_proj.bias"])
        v = F.linear(y, sd[p + "self_attn.v_proj.weight"], sd[p + "self_attn.v_proj.bias"])
        q, k, v = (t.view(B, L, H, d).transpose(1, 2) for t in (q, k, v))
        w = torch.softmax(q @ k.transpose(-1, -2) + causal, dim=-1)
        o = (w @ v).transpose(1, 2).reshape(B, L, C)
        h = h + F.linear(o, sd[p + "self_attn.out_proj.weight"], sd[p + "self_attn.out_proj.bias"])
        y = F.layer_norm(h, (C,), sd[p + "layer_norm2.weight"], sd[p + "layer_norm2.bias"], cfg.layer_norm_eps)
        m = _act(F.linear(y, sd[p + "mlp.fc1.weight"], sd[p + "mlp.fc1.bias"]), cfg.hidden_act)
        h = h + F.linear(m, sd[p + "mlp.fc2.weight"], sd[p + "mlp.fc2.bias"])
    last = F.layer_norm(h, (C,), sd["text_model.final_layer_norm.weight"], sd["text_model.final_layer_norm.bias"],
                        cfg.layer_norm_eps)
    eos = (input_ids == cfg.eos_token_id).int().argmax(dim=-1)              # first EOS (transformers >= 4.30 rule)
    return last, last[torch.arange(B), eos]
