"""GPT-2 (Radford et al. 2019) whose every second MLP is a mixture of experts; ``gpt2_medium_moe8_config()`` = 24 layers,
d_model 1024, 16 heads, 8 experts (BASELINE config 5)."""
from dataclasses import dataclass

import torch
import torch.nn as nn
import torch.nn.functional as F

from ..parallel.moe import MoE


@dataclass
class GPT2MoEConfig:
    vocab_size: int = 50257
    n_positions: int = 1024
    n_embd: int = 768
    n_layer: int = 12
    n_head: int = 12
    num_experts: int = 8          # total experts; num_local_experts = num_experts // world_size
    moe_every: int = 2            # MoE MLP in layers i where i % moe_every == 1
    top_k: int = 1
    capacity_factor: float = 1.0
    dropout: float = 0.0


def gpt2_medium_moe8_config() -> GPT2MoEConfig:
    return GPT2MoEConfig(n_embd=1024, n_layer=24, n_head=16, num_experts=8)


class ExpertMLP(nn.Module):
    grouped_gemm_compatible = True  # fc2(gelu_tanh(fc1(x))): Experts runs all local experts as one wgmma grouped GEMM

    def __init__(self, d):
        super().__init__()
        self.fc1 = nn.Linear(d, 4 * d)
        self.fc2 = nn.Linear(4 * d, d)

    def forward(self, x):
        return self.fc2(F.gelu(self.fc1(x), approximate="tanh"))


class Block(nn.Module):
    def __init__(self, c: GPT2MoEConfig, use_moe: bool, world_size: int):
        super().__init__()
        self.nh = c.n_head
        self.ln1 = nn.LayerNorm(c.n_embd)
        self.qkv = nn.Linear(c.n_embd, 3 * c.n_embd)
        self.proj = nn.Linear(c.n_embd, c.n_embd)
        self.ln2 = nn.LayerNorm(c.n_embd)
        self.use_moe = use_moe
        if use_moe:
            self.mlp = MoE(c.n_embd, ExpertMLP(c.n_embd), num_local_experts=max(1, c.num_experts // world_size), k=c.top_k,
                           capacity_factor=c.capacity_factor)
        else:
            self.mlp = ExpertMLP(c.n_embd)

    def forward(self, x):
        B, S, H = x.shape
        q, k, v = self.qkv(self.ln1(x)).view(B, S, 3, self.nh, H // self.nh).permute(2, 0, 3, 1, 4)
        a = F.scaled_dot_product_attention(q, k, v, is_causal=True).transpose(1, 2).reshape(B, S, H)
        x = x + self.proj(a)
        if self.use_moe:
            y, l_aux, _ = self.mlp(self.ln2(x))
            return x + y, l_aux
        return x + self.mlp(self.ln2(x)), None


class GPT2MoE(nn.Module):
    def __init__(self, c: GPT2MoEConfig, world_size: int = 1):
        super().__init__()
        self.config = c
        self.wte = nn.Embedding(c.vocab_size, c.n_embd)
        self.wpe = nn.Embedding(c.n_positions, c.n_embd)
        self.blocks = nn.ModuleList([Block(c, c.moe_every > 0 and i % c.moe_every == 1, world_size) for i in range(c.n_layer)])
        self.ln_f = nn.LayerNorm(c.n_embd)
        for m in self.modules():
            if isinstance(m, (nn.Linear, nn.Embedding)):
                nn.init.normal_(m.weight, std=0.02)

    def forward(self, idx, targets=None, aux_weight: float = 0.01):
        B, S = idx.shape
        x = self.wte(idx) + self.wpe(torch.arange(S, device=idx.device))
        aux = 0.0
        for blk in self.blocks:
            x, l = blk(x)
            if l is not None:
                aux = aux + l
        logits = F.linear(self.ln_f(x), self.wte.weight)
        if targets is None:
            return logits
        loss = F.cross_entropy(logits.float().view(-1, logits.size(-1)), targets.view(-1))
        return loss + aux_weight * aux, logits
