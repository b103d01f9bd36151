"""Host-side mirror of rten-generate's `Generator` (rten-generate/src/generator.rs) for decoder models whose KV cache
lives in HBM.

The reference drives a `Model` through named tensors -- `input_ids`, `attention_mask`, `position_ids`,
`past_key_values.N.key|value` in, `logits`, `present.N.key|value` out (the Optimum export convention,
`ModelInputsConfig::default()`, generator.rs:270-316) -- keeps the returned `present.*` tensors as the next step's
`past_key_values.*` (:858-886) and doubles a cache's capacity when it is full.  Here the same contract is spoken by
`GPT2DecoderModel`: the cache tensors that cross the `run` boundary are `KvCacheHandle`s (device buffers + valid length),
so nothing is copied per step; capacity doubles the same way.  `Generator` itself only sees names.
"""
from __future__ import annotations

import re
from dataclasses import dataclass
from typing import Callable, Dict, List, Optional, Sequence

import numpy as np

from . import ops as O
from .graphs import GPT2Int8Runner, GPT2Int8Spec


@dataclass
class KvCacheHandle:
    """A `[batch, heads, seq, head]` cache tensor resident in HBM: the buffer, how many positions are valid, how many fit."""
    tensor: O.DeviceTensor
    seq_len: int
    capacity: int
    transposed: bool = False  # stored [batch, heads, head, capacity] (the value cache of this backend)

    @property
    def shape(self):
        b, h = self.tensor.shape[0], self.tensor.shape[1]
        d = self.tensor.shape[2] if self.transposed else self.tensor.shape[3]
        return (b, h, self.seq_len, d)

    def has_capacity(self, n: int) -> bool:
        return n <= self.capacity


# (input prefix, input suffix) -> (output prefix, output suffix), matched in order (generator.rs:283-316)
KV_CACHE_PATTERNS = [(("past_key_values.", ".decoder.key"), ("present.", ".decoder.key")),
                     (("past_key_values.", ".decoder.value"), ("present.", ".decoder.value")),
                     (("past_key_values.", ".key"), ("present.", ".key")),
                     (("past_key_values.", ".value"), ("present.", ".value"))]


class GPT2DecoderModel:
    """GPT-2 small int8 behind the Optimum I/O names.  `run(inputs, outputs)` executes ONE model call: a prompt block of T
    tokens through the operator list, or -- one token per sequence, cache primed -- the captured decode graph (fused
    skinny-M kernels).  The KV cache is owned here and handed out as `present.N.*` handles."""

    def __init__(self, ctx: O.Context, spec: GPT2Int8Spec, batch: int, initial_capacity: int = 64, use_graph: bool = True):
        self.ctx, self.spec, self.batch, self.use_graph = ctx, spec, batch, use_graph
        self.runner = GPT2Int8Runner(ctx, spec, batch, initial_capacity)
        n = len(spec.layers)
        self.input_names = ["input_ids", "attention_mask", "position_ids"] + [f"past_key_values.{i}.{kv}" for i in range(n) for kv in ("key", "value")]
        self.output_names = ["logits"] + [f"present.{i}.{kv}" for i in range(n) for kv in ("key", "value")]
        self._graph_capacity = None

    # -- cache growth: double the capacity, keep the contents (KvCacheData::clone_with_capacity, generator.rs:878-884)
    def _grow(self, needed: int):
        r, ctx = self.runner, self.ctx
        new_cap = r.max_seq
        while new_cap < needed:
            new_cap *= 2
        B, nh, dh, old = r.B, self.spec.heads, self.spec.hidden // self.spec.heads, r.max_seq
        for d in r.layers:
            k2 = ctx.to_device(np.zeros((B, nh, new_cap, dh), np.float32))
            v2 = ctx.to_device(np.zeros((B, nh, dh, new_cap), np.float32))
            if r.past:
                k2.view((B, nh, r.past, dh), (nh * new_cap * dh, new_cap * dh, dh, 1)).assign(
                    d["k"].view((B, nh, r.past, dh), (nh * old * dh, old * dh, dh, 1)))
                v2.view((B, nh, dh, r.past), (nh * dh * new_cap, dh * new_cap, new_cap, 1)).assign(
                    d["vt"].view((B, nh, dh, r.past), (nh * dh * old, dh * old, old, 1)))
            d["k"], d["vt"] = k2, v2
        r.max_seq = new_cap
        self._graph_capacity = None  # the captured decode step addresses the old buffers

    def _handles(self):
        r = self.runner
        out = {}
        for i, d in enumerate(r.layers):
            out[f"present.{i}.key"] = KvCacheHandle(d["k"], r.past, r.max_seq)
            out[f"present.{i}.value"] = KvCacheHandle(d["vt"], r.past, r.max_seq, transposed=True)
        return out

    def run(self, inputs: Dict[str, object], outputs: Sequence[str]) -> Dict[str, object]:
        r = self.runner
        ids = np.ascontiguousarray(inputs["input_ids"], np.int32)
        B, T = ids.shape
        if B != self.batch:
            raise O.OpError(3, f"input_ids batch {B} != model batch {self.batch}")
        past = 0
        for name, v in inputs.items():
            if name.startswith("past_key_values.") and v is not None:
                if not isinstance(v, KvCacheHandle) or v.seq_len != r.past:
                    raise O.OpError(5, f"{name}: not the cache handle of the previous step")
                past = v.seq_len
        if past == 0 and r.past:
            r.reset()  # a new sequence
        if "position_ids" in inputs and inputs["position_ids"] is not None:
            pos = np.asarray(inputs["position_ids"]).reshape(-1, T)
            if not (pos == np.arange(past, past + T)[None, :]).all():
                raise O.OpError(6, "position_ids other than past .. past + T are not supported")
        if "attention_mask" in inputs and inputs["attention_mask"] is not None and not np.asarray(inputs["attention_mask"]).all():
            raise O.OpError(6, "padded sequences (zeros in attention_mask) are not supported")
        if r.past + T > r.max_seq:
            self._grow(r.past + T)
        if T == 1 and r.past > 0 and self.use_graph:
            if self._graph_capacity != r.max_seq:
                r.build_decode_graph()
                self._graph_capacity = r.max_seq
            logits = r.decode_step(ids)
        else:
            logits = r.forward(ids)
        res = {"logits": logits}
        res.update(self._handles())
        return {k: res[k] for k in outputs}


def grow_capacity(capacity: int, needed: int) -> int:
    """The capacity a cache of `capacity` positions grows to so that it holds `needed`: doubled until it does
    (KvCacheData::clone_with_capacity, generator.rs:878-884)"""
    capacity = max(int(capacity), 1)
    while capacity < needed:
        capacity *= 2
    return capacity


class ModelDecoder:
    """A loaded `Model` (an onnxruntime-genai / Optimum decoder export) behind the contract `Generator` speaks, the one
    GPT2DecoderModel speaks: `input_names`, `output_names`, `run(inputs, outputs) -> dict`.  The KV caches are
    KvCacheHandles passed to the model as writable inputs with spare capacity, so the attention nodes append the new
    positions in place instead of copying the past every step.  The first step gets empty caches
    [batch, kv_heads, 0, head] (kv_heads and the head size from the file's declared input dims) of capacity
    `kv_cache_capacity` (or 1).  After each step a cache that cannot take one more position is re-allocated with twice
    the length and its valid prefix copied (one copy launch per cache), as generator.rs:878-884 does."""

    def __init__(self, model, batch: int, kv_cache_capacity: Optional[int] = None):
        self.model, self.ctx, self.batch = model, model.ctx, batch
        self.capacity = max(int(kv_cache_capacity or 1), 1)
        self.input_names, self.output_names = list(model.input_names), list(model.output_names)
        dims = {v["name"]: v["dims"] for v in model.summary["inputs"]}
        self.kv_dims = {}
        for n in self.input_names:
            if n.startswith("past_key_values."):
                d = dims.get(n, [])
                if len(d) != 4 or d[1] <= 0 or d[3] <= 0:
                    raise ValueError(f"{n}: the file does not declare [batch, kv_heads, seq, head] with known kv_heads and head")
                self.kv_dims[n] = (int(d[1]), int(d[3]))

    def _empty(self, name: str) -> KvCacheHandle:
        h, d = self.kv_dims[name]
        return KvCacheHandle(self.ctx.empty((self.batch, h, self.capacity, d)), 0, self.capacity)

    def _with_room(self, c) -> KvCacheHandle:
        """`c` (a handle, or a new present tensor) as a handle that holds one more position"""
        if not isinstance(c, KvCacheHandle):
            c = KvCacheHandle(c, c.shape[2], c.shape[2])
        if c.has_capacity(c.seq_len + 1):
            return c
        cap = grow_capacity(c.capacity, c.seq_len + 1)
        B, H, _, D = c.shape
        t = self.ctx.empty((B, H, cap, D))
        if c.seq_len:
            src = c.tensor.view((B, H, c.seq_len, D), c.tensor.strides)
            t.view((B, H, c.seq_len, D), t.strides).assign(src)
        return KvCacheHandle(t, c.seq_len, cap)

    def run(self, inputs: Dict[str, object], outputs: Sequence[str]) -> Dict[str, object]:
        feeds = {}
        for n, v in inputs.items():
            if n not in self.input_names:
                continue
            if n in self.kv_dims and v is None:
                v = self._empty(n)
            feeds[n] = v
        got = dict(zip(outputs, self.model.run(feeds, list(outputs))))
        for n, v in got.items():
            if n.startswith("present."):
                got[n] = self._with_room(v)
        if "logits" in got and got["logits"].ndim == 3:  # the last position's logits [batch, vocab], as Generator samples
            lg = got["logits"]
            got["logits"] = lg.view((lg.shape[0], lg.shape[2]), (lg.strides[0], lg.strides[2]), (lg.shape[1] - 1) * lg.strides[1])
        return got


class ArgMaxSampler:
    """rten-generate/src/sampler.rs ArgMax: the greedy choice (ties -> lowest id)."""

    def sample(self, logits: np.ndarray) -> np.ndarray:
        return logits.argmax(-1).astype(np.int32)

    def can_sample_device(self, logits: O.DeviceTensor) -> bool:
        return True

    def sample_device(self, logits: O.DeviceTensor) -> np.ndarray:
        """`sample` of device-resident `[batch, vocab]` logits (any strides): TopK with k = 1 on the GPU -- the first
        maximum, or the first NaN, as np.argmax -- and B indices copied back."""
        _, idx = O.TopK(axis=-1).run(logits.ctx, logits, 1)
        return idx.numpy()[:, 0].astype(np.int32)


class TopKSampler:
    """rten-generate/src/sampler.rs TopK: sample from the softmax of the k largest logits / temperature (seeded)."""

    def __init__(self, k: int, temperature: float = 1.0, seed: int = 0):
        self.k, self.temperature, self.rng = k, temperature, np.random.default_rng(seed)

    def sample(self, logits: np.ndarray) -> np.ndarray:
        idx = np.argsort(-logits, axis=-1)[:, :self.k]
        return self._draw(np.take_along_axis(logits, idx, -1), idx)

    def can_sample_device(self, logits: O.DeviceTensor) -> bool:
        """TopK on the device takes k up to TOPK_MAX_K (2048) and at most the vocabulary; any other k samples on the
        host, as before"""
        return 0 < self.k <= min(O.TOPK_MAX_K, logits.shape[-1])

    def sample_device(self, logits: O.DeviceTensor) -> np.ndarray:
        """`sample` of device-resident `[batch, vocab]` logits (any strides): TopK(k) on the GPU, B x k values and
        indices copied back, then the same temperature, softmax and draws as `sample`.  The tokens and the random stream
        are those of `sample` wherever its result is determined: no NaN and no ties among the k + 1 largest logits of a
        row (argsort's order among ties is unspecified; TopK takes the lowest index)."""
        vals, idx = O.TopK(axis=-1).run(logits.ctx, logits, self.k)
        return self._draw(vals.numpy(), idx.numpy())

    def _draw(self, vals: np.ndarray, idx: np.ndarray) -> np.ndarray:
        top = vals / self.temperature
        p = np.exp(top - top.max(-1, keepdims=True))
        p /= p.sum(-1, keepdims=True)
        pick = [self.rng.choice(self.k, p=row) for row in p]
        return idx[np.arange(len(pick)), pick].astype(np.int32)


class Generator:
    """`Generator::from_model` ... iterate (generator.rs:481-1000): every `next()` runs the model once -- the whole prompt
    the first time, then one token per sequence -- and yields the sampled token ids `[batch]`."""

    def __init__(self, model):
        self.model = model
        ins, outs = set(model.input_names), set(model.output_names)
        for need in ("input_ids",):
            if need not in ins:
                raise ValueError(f"model has no '{need}' input")
        if "logits" not in outs:
            raise ValueError("model has no 'logits' output")
        # pair KV-cache inputs with outputs by the name patterns, in pattern order (from_model_config, :493-640)
        self.kv_pairs: List[tuple] = []
        claimed = set()
        for (ip, isf), (op, osf) in KV_CACHE_PATTERNS:
            for name in model.input_names:
                if name in claimed or not (name.startswith(ip) and name.endswith(isf)):
                    continue
                layer = name[len(ip):len(name) - len(isf)]
                if not re.fullmatch(r"\d+", layer):
                    continue
                out_name = f"{op}{layer}{osf}"
                if out_name not in outs:
                    raise ValueError(f"missing output '{out_name}' for KV-cache input '{name}'")
                self.kv_pairs.append((name, out_name))
                claimed.add(name)
        self.kv_cache: Dict[str, Optional[KvCacheHandle]] = {i: None for i, _ in self.kv_pairs}
        self._prompt: Optional[np.ndarray] = None
        self._tokens: List[np.ndarray] = []
        self._seq_len = 0
        self.sampler = ArgMaxSampler()
        self.logits_filters: List[Callable[[np.ndarray, np.ndarray], np.ndarray]] = []
        self._last_logits: Optional[np.ndarray] = None
        self._last_device = None  # the step's device logits, until last_logits copies them

    @property
    def last_logits(self) -> Optional[np.ndarray]:
        """The logits the last step sampled from, `[batch, vocab]` on the host (after the logits filters).  Without
        filters the step samples on the device; the logits are then copied here on first access."""
        if self._last_logits is None and self._last_device is not None:
            self._last_logits = self._last_device.numpy()
            self._last_device = None
        return self._last_logits

    @classmethod
    def from_model(cls, model) -> "Generator":
        return cls(model)

    def with_prompt(self, prompt) -> "Generator":
        self._prompt = np.ascontiguousarray(prompt, np.int32)
        if self._prompt.ndim == 1:
            self._prompt = self._prompt[None, :]
        return self

    def append_prompt(self, prompt):
        p = np.ascontiguousarray(prompt, np.int32)
        p = p[None, :] if p.ndim == 1 else p
        self._prompt = p if self._prompt is None else np.concatenate([self._prompt, p], 1)

    def with_sampler(self, sampler) -> "Generator":
        self.sampler = sampler
        return self

    def with_logits_filter(self, f) -> "Generator":
        self.logits_filters.append(f)
        return self

    def prompt(self):
        return self._prompt

    def prev_tokens(self) -> np.ndarray:
        return np.stack(self._tokens, 1) if self._tokens else np.zeros((0, 0), np.int32)

    def kv_cache_len(self) -> Optional[int]:
        for h in self.kv_cache.values():
            if h is not None:
                return h.seq_len
        return None

    def __iter__(self):
        return self

    def __next__(self) -> np.ndarray:
        if self._prompt is None or self._prompt.shape[1] == 0:
            raise StopIteration
        ids = self._prompt
        B, T = ids.shape
        inputs = {"input_ids": ids}
        if "attention_mask" in self.model.input_names:
            inputs["attention_mask"] = np.ones((B, self._seq_len + T), np.int32)
        if "position_ids" in self.model.input_names:
            inputs["position_ids"] = np.broadcast_to(np.arange(self._seq_len, self._seq_len + T, dtype=np.int32), (B, T))
        inputs.update(self.kv_cache)
        out = self.model.run(inputs, ["logits"] + [o for _, o in self.kv_pairs])
        for i, o in self.kv_pairs:  # the present.* of this step is the past_key_values.* of the next (:858-886)
            self.kv_cache[i] = out[o]
        self._seq_len += T
        dev = out["logits"]
        on_device = (not self.logits_filters and isinstance(dev, O.DeviceTensor) and hasattr(self.sampler, "can_sample_device")
                     and self.sampler.can_sample_device(dev))
        if on_device:
            # sampled on the device: only the picked tokens (and TopK's k candidates) reach the host
            self._last_logits, self._last_device = None, dev
            tok = self.sampler.sample_device(dev)
        else:
            logits = dev.numpy()
            prev = self.prev_tokens()
            for f in self.logits_filters:
                logits = f(logits, prev)
            self._last_logits, self._last_device = logits, None
            tok = self.sampler.sample(logits)
        self._tokens.append(tok)
        self._prompt = tok[:, None]  # next step feeds the sampled token
        return tok
