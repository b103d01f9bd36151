"""Writes the torch-exported decoder fixtures the executor tests load (run once on a CPU machine; the outputs are
committed, and the GPU tests never run the exporter):

  * torch_gpt2.onnx / torch_gpt2.npz: a seeded 2-layer GPT-2-style decoder written the way transformers' GPT2Model /
    GPT2Attention writes it (the c_attn QKV split, the causal `bias` buffer sliced as bias[:, :, kl - ql:kl, :kl],
    where(causal, w, finfo.min), the extended attention mask, position ids from arange(past, past + T), NewGELU, tied
    lm_head).  Inputs input_ids [batch, seq], attention_mask [batch, past + seq], past_key_values.N.key / .value
    [batch, 4, past, 16]; outputs logits, present.N.key / .value.  Batch, seq and past are dynamic axes; the kv-head
    and head dims of the caches stay static, since ModelDecoder reads them from the file's declared input dims.  The
    .npz holds the weights' seed, two feeds (a prompt with a right-padded mask after a non-empty past, and a decode
    step) and each feed's float64 torch outputs.
  * torch_llama_block.onnx / torch_llama_block.npz: transformers' Llama causal-mask construction (without the slice
    assignment `cm[..., :L] = ...`, which exports as ScatterND), rotate_half and repeat_kv, with its feed and float64
    outputs.

The TorchScript exporter (dynamo=False, opset 14) is used.  Its last step inserts onnxscript functions through the
`onnx` package, which this environment does not have; the generator replaces torch's private
`onnx_proto_utils._add_onnxscript_fn` with an identity (these models use no onnxscript functions).

    python tests/golden/make_torch_decoder_fixtures.py"""
import math
import os

import numpy as np
import torch
import torch.nn as nn
from torch.onnx._internal.torchscript_exporter import onnx_proto_utils

HERE = os.path.dirname(os.path.abspath(__file__))
E, H, L, V, NPOS = 64, 4, 2, 128, 64
D = E // H


class Attention(nn.Module):
    def __init__(self):
        super().__init__()
        self.c_attn, self.c_proj = nn.Linear(E, 3 * E), nn.Linear(E, E)
        self.register_buffer("bias", torch.tril(torch.ones((NPOS, NPOS), dtype=torch.bool)).view(1, 1, NPOS, NPOS), persistent=False)

    def _split_heads(self, x):
        return x.view(x.size()[:-1] + (H, D)).permute(0, 2, 1, 3)

    def forward(self, h, past_k, past_v, attention_mask):
        q, k, v = self.c_attn(h).split(E, dim=2)
        q, k, v = self._split_heads(q), self._split_heads(k), self._split_heads(v)
        k = torch.cat((past_k, k), dim=-2)
        v = torch.cat((past_v, v), dim=-2)
        w = torch.matmul(q, k.transpose(-1, -2))
        w = w / torch.full([], v.size(-1) ** 0.5, dtype=w.dtype, device=w.device)
        ql, kl = q.size(-2), k.size(-2)
        causal = self.bias[:, :, kl - ql:kl, :kl]
        mask_value = torch.full([], torch.finfo(w.dtype).min, dtype=w.dtype, device=w.device)
        w = torch.where(causal, w.to(w.dtype), mask_value)
        w = w + attention_mask
        w = nn.functional.softmax(w, dim=-1)
        a = torch.matmul(w, v).permute(0, 2, 1, 3).contiguous()
        a = a.view(a.size()[:-2] + (E,))
        return self.c_proj(a), k, v


def new_gelu(x):
    return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * torch.pow(x, 3.0))))


class Block(nn.Module):
    def __init__(self):
        super().__init__()
        self.ln_1, self.ln_2 = nn.LayerNorm(E), nn.LayerNorm(E)
        self.attn = Attention()
        self.fc, self.proj = nn.Linear(E, 4 * E), nn.Linear(4 * E, E)

    def forward(self, h, past_k, past_v, mask):
        a, k, v = self.attn(self.ln_1(h), past_k, past_v, mask)
        h = h + a
        return h + self.proj(new_gelu(self.fc(self.ln_2(h)))), k, v


class GPT2(nn.Module):
    def __init__(self):
        super().__init__()
        self.wte, self.wpe = nn.Embedding(V, E), nn.Embedding(NPOS, E)
        self.h = nn.ModuleList([Block() for _ in range(L)])
        self.ln_f = nn.LayerNorm(E)

    def forward(self, input_ids, attention_mask, *past):
        past_len = past[0].size(-2)
        pos = torch.arange(past_len, input_ids.size(-1) + past_len, dtype=torch.long, device=input_ids.device).unsqueeze(0)
        h = self.wte(input_ids) + self.wpe(pos)
        mask = attention_mask[:, None, None, :].to(dtype=h.dtype)
        mask = (1.0 - mask) * torch.finfo(h.dtype).min
        presents = []
        for i, blk in enumerate(self.h):
            h, k, v = blk(h, past[2 * i], past[2 * i + 1], mask)
            presents += [k, v]
        logits = torch.matmul(self.ln_f(h), self.wte.weight.t())
        return (logits, *presents)


def llama_mask(attention_mask, x):
    B, T = attention_mask.shape
    causal = torch.full((T, T), torch.finfo(x.dtype).min, dtype=x.dtype, device=x.device)
    causal = torch.triu(causal, diagonal=1)
    causal = causal[None, None, :, :].expand(B, 1, -1, -1)
    padding = attention_mask[:, None, None, :].eq(0)
    return causal.masked_fill(padding, torch.finfo(x.dtype).min)


def rotate_half(x):
    x1 = x[..., : x.shape[-1] // 2]
    x2 = x[..., x.shape[-1] // 2:]
    return torch.cat((-x2, x1), dim=-1)


def repeat_kv(hidden, n_rep):
    b, kv, s, d = hidden.shape
    hidden = hidden[:, :, None, :, :].expand(b, kv, n_rep, s, d)
    return hidden.reshape(b, kv * n_rep, s, d)


class LlamaBlock(nn.Module):
    def forward(self, attention_mask, q, k):
        return llama_mask(attention_mask, q), rotate_half(q), repeat_kv(k, q.shape[1] // k.shape[1])


def gpt2_names():
    ins = ["input_ids", "attention_mask"] + [f"past_key_values.{i}.{kv}" for i in range(L) for kv in ("key", "value")]
    outs = ["logits"] + [f"present.{i}.{kv}" for i in range(L) for kv in ("key", "value")]
    return ins, outs


def gpt2_model(seed=0):
    torch.manual_seed(seed)
    m = GPT2().eval()
    with torch.no_grad():
        for p in m.parameters():
            p.copy_(torch.randn_like(p) * 0.2)
    return m


def gpt2_feeds():
    r = np.random.default_rng(7)
    B = 2
    past = 3
    prompt = dict(input_ids=r.integers(0, V, (B, 5)).astype(np.int64))
    mask = np.ones((B, past + 5), np.int64)
    mask[1, -2:] = 0  # right padding
    prompt["attention_mask"] = mask
    for i in range(L):
        for kv in ("key", "value"):
            prompt[f"past_key_values.{i}.{kv}"] = r.standard_normal((B, H, past, D)).astype(np.float32)
    step = dict(input_ids=r.integers(0, V, (B, 1)).astype(np.int64), attention_mask=np.ones((B, 7), np.int64))
    for i in range(L):
        for kv in ("key", "value"):
            step[f"past_key_values.{i}.{kv}"] = r.standard_normal((B, H, 6, D)).astype(np.float32)
    return {"prompt": prompt, "step": step}


def gpt2_forward_f64(model, feed):
    m = model.double()
    ins, _ = gpt2_names()
    args = [torch.from_numpy(feed[n]) if feed[n].dtype != np.float32 else torch.from_numpy(feed[n]).double() for n in ins]
    with torch.no_grad():
        out = m(*args)
    model.float()
    return [o.numpy() for o in out]


def gpt2_greedy_f64(model, steps):
    """a batch-2 prompt and the `steps` tokens a float64 greedy loop gives from empty caches (ties: the lowest id)"""
    prompt = np.random.default_rng(11).integers(0, V, (2, 4)).astype(np.int64)
    m = model.double()
    ids, past, toks = torch.from_numpy(prompt), [torch.zeros((2, H, 0, D), dtype=torch.float64) for _ in range(2 * L)], []
    total = ids.shape[1]
    with torch.no_grad():
        for _ in range(steps):
            out = m(ids, torch.ones((2, total), dtype=torch.long), *past)
            nxt = out[0][:, -1].argmax(-1)
            toks.append(nxt.numpy())
            past = list(out[1:])
            ids = nxt[:, None]
            total += 1
    model.float()
    return prompt, np.stack(toks, 1).astype(np.int64)


def _export(model, args, path, ins, outs, dynamic_axes):
    saved = onnx_proto_utils._add_onnxscript_fn
    onnx_proto_utils._add_onnxscript_fn = lambda proto, custom_opsets: proto
    try:
        torch.onnx.export(model, args, path, input_names=ins, output_names=outs, dynamic_axes=dynamic_axes, opset_version=14,
                          dynamo=False, do_constant_folding=True)
    finally:
        onnx_proto_utils._add_onnxscript_fn = saved


def main():
    m = gpt2_model()
    ins, outs = gpt2_names()
    feeds = gpt2_feeds()
    f = feeds["prompt"]
    args = tuple(torch.from_numpy(f[n]) for n in ins)
    dyn = {"input_ids": {0: "batch", 1: "seq"}, "attention_mask": {0: "batch", 1: "total"}, "logits": {0: "batch", 1: "seq"}}
    for n in ins[2:] + outs[1:]:
        dyn[n] = {0: "batch", 2: "past"}
    _export(m, args, os.path.join(HERE, "torch_gpt2.onnx"), ins, outs, dyn)
    npz = {}
    for name, feed in feeds.items():
        for k, v in feed.items():
            npz[f"{name}/{k}"] = v
        for k, v in zip(outs, gpt2_forward_f64(m, feed)):
            npz[f"{name}/out/{k}"] = v
    prompt, tokens = gpt2_greedy_f64(m, 8)
    npz["greedy/prompt"], npz["greedy/tokens"] = prompt, tokens
    np.savez_compressed(os.path.join(HERE, "torch_gpt2.npz"), **npz)

    r = np.random.default_rng(9)
    mask = np.ones((2, 6), np.int64)
    mask[1, 4:] = 0
    q = r.standard_normal((2, 4, 6, 8)).astype(np.float32)
    k = r.standard_normal((2, 2, 6, 8)).astype(np.float32)
    blk = LlamaBlock()
    _export(blk, (torch.from_numpy(mask), torch.from_numpy(q), torch.from_numpy(k)), os.path.join(HERE, "torch_llama_block.onnx"),
            ["attention_mask", "q", "k"], ["mask", "rot", "kv"], None)
    with torch.no_grad():
        mo, ro, ko = blk(torch.from_numpy(mask), torch.from_numpy(q).double(), torch.from_numpy(k).double())
    np.savez_compressed(os.path.join(HERE, "torch_llama_block.npz"), attention_mask=mask, q=q, k=k, mask_out=mo.numpy(),
                        rot_out=ro.numpy(), kv_out=ko.numpy())


if __name__ == "__main__":
    main()
