"""rten_b200 -- sm_90a (H100) operator execution backend for the RTen hot path.

The product is `librten_b200.so` (hand-written CUDA behind the C ABI in include/rten_b200.h);
`rten_b200.ops` is the host-side mirror of RTen's operator interface used by the tests, the model
runners and bench.py.  There is no CPU implementation in this package."""
from . import _lib  # noqa: F401
from .ops import (  # noqa: F401
    ACT_GELU, ACT_GELU_TANH, ACT_HARD_SIGMOID, ACT_HARD_SWISH, ACT_NONE, ACT_RELU, ACT_SIGMOID, ACT_SILU, Abs, Add, AddSoftmax, ArgMax, ArgMin, Attention, AveragePool, BatchNormalization, Clip, Concat, Comm, Context, Conv, ConvInteger, ConvIntegerToFloat,
    ConvTranspose, DeviceTensor, Div, DynamicQuantizeLinear, Erf, Exp, FusedMatMul, GatherRows, Gelu, Gemm, GlobalAveragePool, GroupNorm, GroupQueryAttention, GRU, HardSigmoid, HardSwish, InstanceNormalization,
    LayerNormalization, LSTM, MatMul, MatMulInteger, MatMulIntegerToFloat, MatMulNBits, MaxPool, Mul, MultiHeadAttention, Neg, OpError, Packed, Pow, QuantizedLinear, Reciprocal, ReduceMean, ReduceSum, Relu, Resize, RMSNormalization, RotaryEmbedding, ScatterRows, Sigmoid,
    SimplifiedLayerNormalization, Silu, SkipLayerNormalization, SkipSimplifiedLayerNormalization, Softmax, Sqrt, Sub, Tanh, TopK, Upsample, from_torch,
)
from .ops import (  # noqa: F401
    And, Equal, Expand, Greater, GreaterOrEqual, Less, LessOrEqual, Not, Or, Slice, Split, Trilu, Where, Xor,
)
