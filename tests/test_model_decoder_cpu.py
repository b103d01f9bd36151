"""CPU-only: ModelDecoder's cache capacity arithmetic against a fake model and fake device tensors -- the first step's
empty caches, when a cache is re-allocated, to what capacity, and how many positions are copied."""
import numpy as np

from rten_b200.generate import KvCacheHandle, ModelDecoder, grow_capacity


class FakeTensor:
    def __init__(self, log, shape, strides=None):
        self.log, self.shape = log, tuple(shape)
        self.strides = strides or tuple(int(np.prod(self.shape[i + 1:])) for i in range(len(self.shape)))
        self.ndim = len(self.shape)

    def view(self, shape, strides, offset=0):
        return FakeTensor(self.log, shape, strides)

    def assign(self, src):
        self.log.append(("copy", src.shape[2]))


class FakeCtx:
    def __init__(self):
        self.log = []

    def empty(self, shape, dtype=np.float32):
        self.log.append(("alloc", shape[2]))
        return FakeTensor(self.log, shape)


class FakeModel:
    """past_key_values.0.key / value [batch, 2, seq, 8] in; present.0.* out, each the past handle grown by the step's
    tokens, or a new tensor when the handle has no room (the executor's fallback)"""

    def __init__(self):
        self.ctx = FakeCtx()
        self.input_names = ["input_ids", "attention_mask", "past_key_values.0.key", "past_key_values.0.value"]
        self.output_names = ["logits", "present.0.key", "present.0.value"]
        self.summary = {"inputs": [{"name": n, "dims": [-1, 2, -1, 8]} for n in self.input_names[2:]]}

    def run(self, feeds, outputs):
        T = feeds["input_ids"].shape[1]
        res = {"logits": FakeTensor(self.ctx.log, (1, T, 5))}
        for kv in ("key", "value"):
            h = feeds[f"past_key_values.0.{kv}"]
            n = h.seq_len + T
            res[f"present.0.{kv}"] = KvCacheHandle(h.tensor, n, h.capacity) if n <= h.capacity else FakeTensor(self.ctx.log, (1, 2, n, 8))
        return [res[o] for o in outputs]


def test_grow_capacity():
    assert [grow_capacity(c, n) for c, n in ((1, 1), (1, 2), (3, 4), (4, 4), (6, 13), (0, 3))] == [1, 2, 6, 4, 24, 4]


def _steps(capacity, prompt, steps):
    m = FakeModel()
    dec = ModelDecoder(m, 1, capacity)
    assert dec.kv_dims == {"past_key_values.0.key": (2, 8), "past_key_values.0.value": (2, 8)}
    past, seen = {"past_key_values.0.key": None, "past_key_values.0.value": None}, []
    ids = np.zeros((1, prompt), np.int32)
    for _ in range(steps):
        out = dec.run(dict(input_ids=ids, attention_mask=None, **past), m.output_names)
        assert out["logits"].shape == (1, 5)
        k = out["present.0.key"]
        seen.append((k.seq_len, k.capacity))
        past = {"past_key_values.0.key": k, "past_key_values.0.value": out["present.0.value"]}
        ids = np.zeros((1, 1), np.int32)
    return seen, m.ctx.log


def test_capacity_that_fits():
    seen, log = _steps(64, 3, 6)
    assert seen == [(3 + i, 64) for i in range(6)]
    assert log == [("alloc", 64), ("alloc", 64)]  # the two empty caches; nothing is re-allocated or copied


def test_capacity_one_doubles():
    seen, log = _steps(None, 3, 10)
    assert seen == [(3, 6), (4, 6), (5, 6), (6, 12), (7, 12), (8, 12), (9, 12), (10, 12), (11, 12), (12, 24)]
    # empty caches of 1; the prompt's new caches (3 positions) re-allocated to 6 with 3 copied; then 6 -> 12 and 12 -> 24
    assert log == [("alloc", 1), ("alloc", 1)] + [("alloc", 6), ("copy", 3)] * 2 + [("alloc", 12), ("copy", 6)] * 2 + \
        [("alloc", 24), ("copy", 12)] * 2
