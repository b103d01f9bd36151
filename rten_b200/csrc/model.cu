// Minimal graph executor behind the C ABI (include/rten_b200.h: rten_b200_model_*): what RTen's `Model::load` +
// `Graph::run_plan` do around the operators of this library (src/model.rs, src/graph.rs:880-1286), restated for the
// hot-path operator set:
//   load : ONNX bytes -> nodes + initialisers (onnx_reader.cu; int64 tensors become i32 like rten's loader does) ->
//          constants uploaded to HBM once -> load-time fusions (Mul(x, Sigmoid(x)) -> Silu, then Conv + activation
//          and MatMul + Add(bias): the subset of src/optimize.rs the models need) -> weights prepacked once
//          (`Operator::prepack`, src/graph.rs:488-565).
//   run  : the nodes in topological (file) order, one C-ABI operator call each; temporaries are reference counted and
//          returned to the context pool after their last consumer (src/graph.rs:1100-1180); an operator that can run in
//          place does so when the executor holds the last reference to its input (src/graph.rs:973-1049); shape-only
//          operators (Reshape, Flatten, Squeeze, Unsqueeze, Transpose, Identity) are views -- no kernel, no copy.
//          A Concat over the channels of NCHW tensors is written in place by its producers where the load found that
//          possible (plan_concat_elision): the first such producer to run allocates the Concat's buffer and every one of
//          them gets a strided view of its channel slice as `out`, so the Concat node copies only the other inputs --
//          nothing when there are none.  RTEN_B200_NO_CONCAT_ELISION=1 (read at load) turns that off for comparisons.
// Operators: Conv, ConvInteger, ConvTranspose (without output_shape), Relu, Clip, Sigmoid, HardSigmoid, HardSwish,
// MaxPool, AveragePool (ceil_mode 0), GlobalAveragePool, ReduceMean, Resize and Upsample (constant scales / sizes), Concat, Gemm, MatMul, MatMulInteger, MatMulNBits
// (com.microsoft), Add, Mul, Softmax, LayerNormalization, RMSNormalization, SimplifiedLayerNormalization,
// SkipLayerNormalization and SkipSimplifiedLayerNormalization (com.microsoft, outputs 0 and 3), Gelu, Erf, Gather, Cast,
// DynamicQuantizeLinear, Attention, RotaryEmbedding, GroupQueryAttention and MultiHeadAttention (com.microsoft, three outputs), GRU and LSTM, Constant and
// the view operators.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <set>
#include <string>
#include <vector>

#include "api_shared.h"
#include "api_util.h"
#include "onnx_reader.h"
#include "rowops.h"

using namespace rtb;

namespace {

enum ValueKind { V_UNSET = 0, V_CONST, V_INPUT, V_TEMP };

struct ValueSlot {
    std::string name;
    ValueKind kind = V_UNSET;
    rten_tensor t{};
    bool has_host_ints = false;       // shape-like constant (int64 in the file): usable by Reshape / axes inputs
    std::vector<int64_t> host_ints;
    bool has_host_floats = false;     // small f32 constant: usable as the scales of Resize / Upsample
    std::vector<float> host_floats;
    // run state
    int root = -1;        // value that owns the allocation (self for owners)
    int pending = 0;      // consumers still to run
    int views = 0;        // live views of this owner
    bool live = false;
    bool owned = false;   // allocation belongs to the executor (pool)
};

struct OpNode {
    onnx::Node n;
    std::vector<int> in, out;  // value ids (-1 = absent optional input)
    rten_packed* packed = nullptr;
    rten_activation activation = {RTEN_ACT_NONE, 0.0f, 0.0f};  // fused activation of a Conv
    int bias_value = -1;       // fused Add(bias) of a MatMul
    // Concat elision (plan_concat_elision).  On a Concat: the channel count of every input and whether its producer
    // writes it in place.  On a producer: the Concat node and the input slot its output is written into.
    std::vector<int64_t> cat_channels;
    std::vector<char> cat_in_place;
    int cat_node = -1, cat_slot = -1;
};

}  // namespace

struct rten_model {
    rten_ctx* ctx = nullptr;
    std::vector<ValueSlot> values;
    std::map<std::string, int> by_name;
    std::vector<OpNode> nodes;
    std::vector<int> inputs, outputs;
    std::vector<void*> const_allocs;
    float* one = nullptr;  // device scalar 1.0f (Cast int32 -> float through cast_scale)
    std::string summary;

    int value_id(const std::string& name) {
        if (name.empty()) return -1;
        auto it = by_name.find(name);
        if (it != by_name.end()) return it->second;
        ValueSlot v;
        v.name = name;
        values.push_back(v);
        by_name[name] = (int)values.size() - 1;
        return (int)values.size() - 1;
    }
};

namespace {

rten_status mfail(rten_ctx* ctx, rten_status st, const std::string& msg) {
    if (ctx) ctx->err = msg;
    return st;
}

int dtype_of(int32_t onnx_dt) {
    switch (onnx_dt) {
        case onnx::DT_FLOAT: return RTEN_F32;
        case onnx::DT_INT32: case onnx::DT_INT64: case onnx::DT_BOOL: return RTEN_I32;
        case onnx::DT_INT8: return RTEN_I8;
        case onnx::DT_UINT8: return RTEN_U8;
        default: return -1;
    }
}

// initialiser / Constant tensor -> device constant (int64 narrowed to i32, the only integer width of the path)
rten_status upload_constant(rten_model* m, const onnx::Tensor& t, ValueSlot* v) {
    rten_ctx* ctx = m->ctx;
    const int dt = dtype_of(t.data_type);
    if (dt < 0) return mfail(ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported tensor type in initializer '" + t.name + "'");
    if (t.external) return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "external tensor data is not supported ('" + t.name + "')");
    if ((int)t.dims.size() > RTEN_MAX_DIMS) return mfail(ctx, RTEN_ERR_INVALID_VALUE, "tensor rank out of range");
    const int64_t n = t.numel();
    std::vector<uint8_t> conv;
    const uint8_t* src = t.data.data();
    if (t.data_type == onnx::DT_INT64) {
        conv.resize((size_t)n * 4);
        v->has_host_ints = true;
        v->host_ints.resize((size_t)n);
        for (int64_t i = 0; i < n; i++) {
            int64_t x;
            memcpy(&x, t.data.data() + 8 * i, 8);
            v->host_ints[(size_t)i] = x;
            const int32_t y = (int32_t)std::max<int64_t>(INT32_MIN, std::min<int64_t>(INT32_MAX, x));
            memcpy(conv.data() + 4 * i, &y, 4);
        }
        src = conv.data();
    } else if (t.data_type == onnx::DT_BOOL) {
        conv.resize((size_t)n * 4);
        for (int64_t i = 0; i < n; i++) {
            const int32_t y = t.data[(size_t)i] ? 1 : 0;
            memcpy(conv.data() + 4 * i, &y, 4);
        }
        src = conv.data();
    } else if (t.data_type == onnx::DT_FLOAT && n <= RTEN_MAX_DIMS) {
        v->has_host_floats = true;
        v->host_floats.resize((size_t)n);
        if (n) memcpy(v->host_floats.data(), t.data.data(), (size_t)n * 4);
    } else if (t.data_type == onnx::DT_INT32) {
        v->has_host_ints = true;
        v->host_ints.resize((size_t)n);
        for (int64_t i = 0; i < n; i++) {
            int32_t x;
            memcpy(&x, t.data.data() + 4 * i, 4);
            v->host_ints[(size_t)i] = x;
        }
    }
    const size_t bytes = (size_t)n * dtype_size(dt);
    void* d = nullptr;
    RTB_TRY(pool_alloc(ctx, bytes ? bytes : 16, &d));
    m->const_allocs.push_back(d);
    if (bytes) RTB_CUDA(ctx, cudaMemcpyAsync(d, src, bytes, cudaMemcpyHostToDevice, ctx->stream));
    RTB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // `conv` / the file buffer may go away
    v->kind = V_CONST;
    v->t.data = d;
    v->t.dtype = dt;
    v->t.ndim = (int)t.dims.size();
    for (int i = 0; i < v->t.ndim; i++) v->t.shape[i] = t.dims[(size_t)i];
    set_contiguous(&v->t);
    v->t.device = ctx->device;
    return RTEN_OK;
}

const std::set<std::string>& supported_ops() {
    static const std::set<std::string> s = {
        "Conv", "ConvTranspose", "Relu", "Clip", "Sigmoid", "HardSigmoid", "HardSwish", "MaxPool", "AveragePool", "Resize", "Upsample", "Concat", "GlobalAveragePool", "ReduceMean", "Reshape", "Flatten", "Squeeze", "Unsqueeze", "Transpose",
        "Identity", "Gemm", "MatMul", "Add", "Mul", "Softmax", "LayerNormalization", "Gelu", "Erf", "Gather",
        "DynamicQuantizeLinear", "MatMulInteger", "ConvInteger", "Cast", "Attention", "MatMulNBits", "GroupQueryAttention",
        "MultiHeadAttention", "RotaryEmbedding", "GRU", "LSTM", "Constant", "RMSNormalization", "SimplifiedLayerNormalization",
        "SkipLayerNormalization", "SkipSimplifiedLayerNormalization"};
    return s;
}

// RNN direction attribute (src/op_registry/onnx_registry.rs get_common_rnn_attrs): 0 forward, 1 reverse, 2 bidirectional,
// -1 for any other value
int rnn_direction(const onnx::Node& n) {
    const onnx::Attribute* a = n.attr("direction");
    if (!a) return 0;
    if (a->s == "forward") return 0;
    if (a->s == "reverse") return 1;
    if (a->s == "bidirectional") return 2;
    return -1;
}

// The attributes get_common_rnn_attrs and the GRU / LSTM readers refuse, refused at load with the operator's name
rten_status check_rnn_attrs(rten_ctx* ctx, const onnx::Node& n) {
    const bool gru = n.op_type == "GRU";
    const std::string& op = n.op_type;
    if (!n.attr("hidden_size")) return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, op + ": missing attribute hidden_size");
    const int dir = rnn_direction(n);
    if (dir < 0) return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, op + ": unsupported direction");
    for (const char* name : {"activation_alpha", "activation_beta"}) {
        const onnx::Attribute* a = n.attr(name);
        if (a && !a->floats.empty()) return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, op + ": " + name + " is not supported");
    }
    if (const onnx::Attribute* a = n.attr("activations")) {
        const std::vector<std::string> dflt = gru ? std::vector<std::string>{"Sigmoid", "Tanh"}
                                                  : std::vector<std::string>{"Sigmoid", "Tanh", "Tanh"};
        bool ok = a->strings.empty();
        if (!ok && a->strings.size() == dflt.size() * (dir == 2 ? 2 : 1)) {
            ok = true;
            for (size_t i = 0; i < a->strings.size(); i++) ok = ok && a->strings[i] == dflt[i % dflt.size()];
        }
        if (!ok) return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, op + ": only the default activations are supported");
    }
    if (n.attr_f("clip", 0.0f) != 0.0f) return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, op + ": clip is not supported");
    if (n.attr_i("layout", 0) != 0) return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, op + ": layout = 1 is not supported");
    if (!gru && n.attr_i("input_forget", 0) != 0)
        return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, op + ": input_forget is not supported");
    if (!gru && n.inputs.size() > 7 && !n.inputs[7].empty())
        return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, op + ": peephole weights (input 7) are not supported");
    return RTEN_OK;
}

bool is_view_op(const std::string& op) {
    return op == "Reshape" || op == "Flatten" || op == "Squeeze" || op == "Unsqueeze" || op == "Transpose" || op == "Identity";
}
bool is_in_place_op(const std::string& op) {
    return op == "Relu" || op == "Clip" || op == "Gelu" || op == "Erf" || op == "Softmax" || op == "Sigmoid" || op == "Silu" ||
           op == "HardSigmoid" || op == "HardSwish";
}

// HardSigmoid's attributes with the reference's defaults (src/op_registry/onnx_registry.rs:1228-1232)
float hard_sigmoid_alpha(const onnx::Node& n) { return n.attr_f("alpha", 0.2f); }
float hard_sigmoid_beta(const onnx::Node& n) { return n.attr_f("beta", 0.5f); }

// The activation node `n` as a fused Conv epilogue, or RTEN_ACT_NONE for any other node (Clip is not fused)
rten_activation conv_activation(const onnx::Node& n) {
    const std::string& op = n.op_type;
    if (op == "Relu") return {RTEN_ACT_RELU, 0.0f, 0.0f};
    if (op == "Sigmoid") return {RTEN_ACT_SIGMOID, 0.0f, 0.0f};
    if (op == "Silu") return {RTEN_ACT_SILU, 0.0f, 0.0f};
    if (op == "HardSigmoid") return {RTEN_ACT_HARD_SIGMOID, hard_sigmoid_alpha(n), hard_sigmoid_beta(n)};
    if (op == "HardSwish") return {RTEN_ACT_HARD_SWISH, 0.0f, 0.0f};
    return {RTEN_ACT_NONE, 0.0f, 0.0f};
}

// Resize / Upsample attributes as the reference reads them (src/op_registry/onnx_registry.rs:1721-1778, 1789-1810):
// antialias, exclude_outside, extrapolation_value, keep_aspect_ratio_policy and cubic_coeff_a must have their defaults;
// `cubic` falls back to linear; defaults nearest, round_prefer_floor, half_pixel.  Upsample is always asymmetric + floor
// (src/ops/resize.rs:629-642).
rten_status fill_resize_params(rten_ctx* ctx, const onnx::Node& n, rten_resize_params* p) {
    memset(p, 0, sizeof(*p));
    const bool upsample = n.op_type == "Upsample";
    auto str = [&](const char* name, const char* dflt) {
        const onnx::Attribute* a = n.attr(name);
        return a ? a->s : std::string(dflt);
    };
    const std::string mode = str("mode", "nearest");
    if (mode == "nearest") p->mode = RTEN_RESIZE_NEAREST;
    else if (mode == "linear" || (mode == "cubic" && !upsample)) p->mode = RTEN_RESIZE_LINEAR;
    else return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, n.op_type + ": unsupported mode '" + mode + "'");
    if (upsample) {
        p->coord_mode = RTEN_RESIZE_ASYMMETRIC;
        p->nearest_mode = RTEN_RESIZE_FLOOR;
        return RTEN_OK;
    }
    if (n.attr_i("antialias", 0) != 0) return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "Resize: antialias must be 0");
    if (n.attr_f("cubic_coeff_a", -0.75f) != -0.75f) return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "Resize: cubic_coeff_a must be -0.75");
    if (n.attr_i("exclude_outside", 0) != 0) return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "Resize: exclude_outside must be 0");
    if (n.attr_f("extrapolation_value", 0.0f) != 0.0f) return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "Resize: extrapolation_value must be 0");
    if (str("keep_aspect_ratio_policy", "stretch") != "stretch")
        return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "Resize: keep_aspect_ratio_policy must be stretch");
    const std::string nm = str("nearest_mode", "round_prefer_floor"), cm = str("coordinate_transformation_mode", "half_pixel");
    if (nm == "floor") p->nearest_mode = RTEN_RESIZE_FLOOR;
    else if (nm == "ceil") p->nearest_mode = RTEN_RESIZE_CEIL;
    else if (nm == "round_prefer_floor") p->nearest_mode = RTEN_RESIZE_ROUND_PREFER_FLOOR;
    else if (nm == "round_prefer_ceil") p->nearest_mode = RTEN_RESIZE_ROUND_PREFER_CEIL;
    else return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "Resize: unsupported nearest_mode '" + nm + "'");
    if (cm == "half_pixel") p->coord_mode = RTEN_RESIZE_HALF_PIXEL;
    else if (cm == "asymmetric") p->coord_mode = RTEN_RESIZE_ASYMMETRIC;
    else if (cm == "align_corners") p->coord_mode = RTEN_RESIZE_ALIGN_CORNERS;
    else if (cm == "pytorch_half_pixel") p->coord_mode = RTEN_RESIZE_PYTORCH_HALF_PIXEL;
    else return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "Resize: unsupported coordinate_transformation_mode '" + cm + "'");
    return RTEN_OK;
}

// MaxPool / AveragePool attributes (kernel_shape, pads, strides)
struct PoolAttrs {
    int32_t kernel[2], pads[4] = {0, 0, 0, 0}, strides[2] = {1, 1};
};
rten_status fill_pool_attrs(rten_ctx* ctx, const onnx::Node& n, PoolAttrs* a) {
    const std::vector<int64_t> k = n.attr_ints("kernel_shape"), pd = n.attr_ints("pads"), sd = n.attr_ints("strides");
    if (k.size() != 2) return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, n.op_type + ": only 2-D kernels are supported");
    a->kernel[0] = (int32_t)k[0];
    a->kernel[1] = (int32_t)k[1];
    for (size_t i = 0; i < pd.size() && i < 4; i++) a->pads[i] = (int32_t)pd[i];
    for (size_t i = 0; i < sd.size() && i < 2; i++) a->strides[i] = (int32_t)sd[i];
    return RTEN_OK;
}

bool writes_concat_in_place(const std::string& op) {
    // The operators whose entry points write a caller's strided `out` directly: every store path of the convolutions
    // takes the output's pixel and channel strides (the TMA store map is built from them, the register epilogues and
    // the depthwise and halo kernels index with them, the explicit-im2col path falls back to a strided copy), the
    // stride phases of ConvTranspose are such views already, and the pooling and Resize kernels index with the output
    // strides.  The elementwise activations are left out: they reach a strided `out` through a temporary and a copy,
    // which costs what the Concat copy costs.  So is a nested Concat, whose buffer would have to exist before its own.
    return op == "Conv" || op == "ConvTranspose" || op == "MaxPool" || op == "AveragePool" || op == "Resize" || op == "Upsample";
}

rten_status fill_conv_params(rten_ctx* ctx, const onnx::Node& n, rten_conv_params* p) {
    memset(p, 0, sizeof(*p));
    const onnx::Attribute* ap = n.attr("auto_pad");
    if (ap && (ap->s == "SAME_UPPER" || ap->s == "SAME_LOWER")) p->auto_pad_same = 1;
    if (ap && ap->s == "SAME_LOWER") return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "auto_pad SAME_LOWER is not supported");
    const std::vector<int64_t> pads = n.attr_ints("pads"), st = n.attr_ints("strides"), dl = n.attr_ints("dilations");
    if (pads.size() == 4) {  // ONNX [top, left, bottom, right]
        for (int i = 0; i < 4; i++) p->pads[i] = (int32_t)pads[(size_t)i];
    } else if (pads.size() == 2) {
        p->pads[0] = (int32_t)pads[0];
        p->pads[1] = (int32_t)pads[1];
    } else if (!pads.empty()) {
        return mfail(ctx, RTEN_ERR_INVALID_VALUE, "Wrong number of pad values");
    }
    p->groups = (int32_t)n.attr_i("group", 1);
    p->n_strides = st.empty() ? 2 : (int32_t)st.size();
    p->n_dilations = dl.empty() ? 2 : (int32_t)dl.size();
    for (int i = 0; i < 2; i++) {
        p->strides[i] = i < (int)st.size() ? (int32_t)st[(size_t)i] : 1;
        p->dilations[i] = i < (int)dl.size() ? (int32_t)dl[(size_t)i] : 1;
    }
    return RTEN_OK;
}

// ConvTranspose attributes as the reference reads them (src/op_registry/onnx_registry.rs:912-972, 1032-1052): strides,
// dilations and pads default to as many values as kernel_shape has spatial axes (none without kernel_shape), auto_pad
// SAME_UPPER / SAME_LOWER is `Padding::Same`, output_padding is absent unless set.
rten_status fill_conv_transpose_params(rten_ctx* ctx, const onnx::Node& n, rten_conv_transpose_params* p) {
    memset(p, 0, sizeof(*p));
    const onnx::Attribute* ap = n.attr("auto_pad");
    if (ap && !ap->s.empty() && ap->s != "NOTSET" && ap->s != "VALID" && ap->s != "SAME_UPPER" && ap->s != "SAME_LOWER")
        return mfail(ctx, RTEN_ERR_INVALID_VALUE, "auto_pad: unsupported value");
    p->auto_pad_same = ap && (ap->s == "SAME_UPPER" || ap->s == "SAME_LOWER");
    const size_t nsp = n.attr_ints("kernel_shape").size();
    // (a count that does not match the input's rank fails in the operator, with the reference's message)
    auto read = [&](const char* name, size_t dflt_len, int32_t dflt, int32_t* dst, size_t cap, int32_t* count) {
        const std::vector<int64_t> v = n.attr(name) ? n.attr_ints(name) : std::vector<int64_t>(dflt_len, dflt);
        for (size_t i = 0; i < v.size() && i < cap; i++) dst[i] = (int32_t)v[i];
        *count = (int32_t)v.size();
    };
    read("strides", nsp, 1, p->strides, 2, &p->n_strides);
    read("dilations", nsp, 1, p->dilations, 2, &p->n_dilations);
    read("pads", 2 * nsp, 0, p->pads, 4, &p->n_pads);
    if (n.attr("output_padding")) read("output_padding", 0, 0, p->output_padding, 2, &p->n_output_padding);
    p->groups = (int32_t)n.attr_i("group", 1);
    return RTEN_OK;
}

}  // namespace

extern "C" {

rten_status rten_b200_onnx_summary(const void* bytes, size_t len, char* json_out, size_t cap, size_t* needed) {
    onnx::Model m;
    std::string err;
    if (!onnx::decode_model(reinterpret_cast<const uint8_t*>(bytes), len, &m, &err)) return RTEN_ERR_INVALID_VALUE;
    const std::string s = onnx::summary_json(m);
    if (needed) *needed = s.size() + 1;
    if (json_out && cap) {
        const size_t n = std::min(cap - 1, s.size());
        memcpy(json_out, s.data(), n);
        json_out[n] = 0;
    }
    return RTEN_OK;
}

void rten_b200_model_free(rten_model* m) {
    if (!m) return;
    for (OpNode& n : m->nodes)
        if (n.packed) rten_b200_packed_free(m->ctx, n.packed);
    for (void* p : m->const_allocs) pool_free(m->ctx, p);
    delete m;
}

rten_status rten_b200_model_load(rten_ctx* ctx, const void* bytes, size_t len, rten_model** out) {
    if (!ctx || !out || (!bytes && len)) return RTEN_ERR_INVALID_VALUE;
    *out = nullptr;
    cudaSetDevice(ctx->device);
    onnx::Model om;
    std::string err;
    if (!onnx::decode_model(reinterpret_cast<const uint8_t*>(bytes), len, &om, &err)) return mfail(ctx, RTEN_ERR_INVALID_VALUE, "ONNX decode failed: " + err);
    if (!om.has_graph) return mfail(ctx, RTEN_ERR_INVALID_VALUE, "ONNX model has no graph");
    std::unique_ptr<rten_model, void (*)(rten_model*)> m(new rten_model(), rten_b200_model_free);
    m->ctx = ctx;
    m->summary = onnx::summary_json(om);
    // constants
    for (const onnx::Tensor& t : om.graph.initializers) {
        const int id = m->value_id(t.name);
        RTB_TRY(upload_constant(m.get(), t, &m->values[(size_t)id]));
    }
    {
        void* d = nullptr;
        RTB_TRY(pool_alloc(ctx, 16, &d));
        m->const_allocs.push_back(d);
        const float one = 1.0f;
        RTB_CUDA(ctx, cudaMemcpy(d, &one, 4, cudaMemcpyHostToDevice));
        m->one = (float*)d;
    }
    for (const onnx::ValueInfo& vi : om.graph.inputs) {
        const int id = m->value_id(vi.name);
        if (m->values[(size_t)id].kind == V_CONST) continue;  // (old exporters list initialisers among the inputs)
        m->values[(size_t)id].kind = V_INPUT;
        m->inputs.push_back(id);
    }
    // nodes (the file order is topological: onnx.proto3 requires it, like src/model.rs relies on)
    for (const onnx::Node& n : om.graph.nodes) {
        if (!n.domain.empty() && n.domain != "ai.onnx" && n.domain != "com.microsoft")
            return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "unsupported operator domain '" + n.domain + "'");
        if (!supported_ops().count(n.op_type)) return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "unsupported operator " + n.op_type);
        if (n.op_type == "Constant") {
            const onnx::Attribute* a = n.attr("value");
            if (!a || !a->has_t || n.outputs.size() != 1) return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "Constant without a tensor value");
            onnx::Tensor t = a->t;
            t.name = n.outputs[0];
            const int id = m->value_id(t.name);
            RTB_TRY(upload_constant(m.get(), t, &m->values[(size_t)id]));
            continue;
        }
        if (n.op_type == "MatMulNBits") {  // src/op_registry/onnx_registry.rs:1376-1402
            if (n.attr_i("bits", 4) != 4) return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "MatMulNBits: only bits = 4 is supported");
            if (!n.attr("block_size")) return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "MatMulNBits: missing attribute block_size");
        }
        if (n.op_type == "GroupQueryAttention") {  // src/op_registry/onnx_registry.rs:1467-1492, contrib.rs:817-821
            if (n.domain != "com.microsoft") return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "unsupported operator GroupQueryAttention");
            if (!n.attr("num_heads") || !n.attr("kv_num_heads"))
                return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "GroupQueryAttention: missing attribute num_heads or kv_num_heads");
            if (n.inputs.size() > 12)
                return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "GroupQueryAttention: quantization and Q/K norm inputs (12-15) are not supported");
        }
        if (n.op_type == "MultiHeadAttention") {  // src/op_registry/onnx_registry.rs:1495-1505, contrib.rs:302-315
            if (n.domain != "com.microsoft") return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "unsupported operator MultiHeadAttention");
            if (!n.attr("num_heads")) return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "MultiHeadAttention: missing attribute num_heads");
            if (n.attr("scale") && !(n.attr_f("scale", 0.0f) > 0.0f))
                return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "MultiHeadAttention: an explicit scale must be positive");
            for (size_t i = 8; i < n.inputs.size(); i++)
                if (!n.inputs[i].empty())
                    return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "MultiHeadAttention: past_sequence_length and cache_indirection (inputs 8, 9) are not supported");
            if (n.outputs.size() > 3 && !n.outputs[3].empty())
                return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "MultiHeadAttention: the qk output (3) is not supported");
        }
        if (n.op_type == "RMSNormalization" || n.op_type == "SimplifiedLayerNormalization") {  // onnx_registry.rs:1584-1590, 1905-1911
            if (n.domain == "com.microsoft") return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "unsupported operator com.microsoft." + n.op_type);
            if (n.attr_i("stash_type", 1) != 1) return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, n.op_type + ": stash_type must be 1");
            for (size_t i = 1; i < n.outputs.size(); i++)
                if (!n.outputs[i].empty())
                    return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, n.op_type + ": only the normalized output (0) is supported");
        }
        if (n.op_type == "SkipLayerNormalization" || n.op_type == "SkipSimplifiedLayerNormalization") {  // onnx_registry.rs:1918-1932
            if (n.domain != "com.microsoft") return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "unsupported operator " + n.op_type);
            if (!n.attr("epsilon")) return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, n.op_type + ": missing attribute epsilon");
            // (the reference returns placeholder zeros for the training statistics, which no inference graph reads)
            for (size_t i = 1; i < 3 && i < n.outputs.size(); i++)
                if (!n.outputs[i].empty())
                    return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, n.op_type + ": the mean and inv_std_var outputs (1, 2) are not supported");
        }
        if (n.op_type == "Resize" || n.op_type == "Upsample") {
            rten_resize_params rp;
            RTB_TRY(fill_resize_params(ctx, n, &rp));
        }
        if (n.op_type == "AveragePool" && n.attr_i("ceil_mode", 0) != 0)
            return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "AveragePool: ceil_mode = 1 is not supported");
        if (n.op_type == "Concat" && !n.attr("axis")) return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "Concat: missing attribute axis");
        if (n.op_type == "GRU" || n.op_type == "LSTM") RTB_TRY(check_rnn_attrs(ctx, n));
        if (n.op_type == "ConvTranspose" && n.attr("output_shape"))  // (the reference does not read it)
            return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "ConvTranspose: the output_shape attribute is not supported");
        if (n.op_type == "RotaryEmbedding" && n.domain == "com.microsoft")
            return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "unsupported operator com.microsoft.RotaryEmbedding");
        OpNode on;
        on.n = n;
        if (n.op_type == "Clip") {
            // legacy (opset < 11) min / max attributes become constant inputs 1 / 2, as the reference's reader does
            // (src/op_registry/onnx_registry.rs:887-898)
            const char* names[2] = {"min", "max"};
            for (int k = 0; k < 2; k++) {
                const onnx::Attribute* a = n.attr(names[k]);
                if (!a) continue;
                onnx::Tensor t;
                t.name = n.name + "/" + (n.outputs.empty() ? std::string() : n.outputs[0]) + "/clip_" + names[k];
                t.data_type = onnx::DT_FLOAT;
                const float v = a->f;
                t.data.resize(4);
                memcpy(t.data.data(), &v, 4);
                const int id = m->value_id(t.name);
                RTB_TRY(upload_constant(m.get(), t, &m->values[(size_t)id]));
                if (on.n.inputs.size() < (size_t)k + 2) on.n.inputs.resize((size_t)k + 2);
                on.n.inputs[(size_t)k + 1] = t.name;
            }
        }
        if (n.op_type == "Upsample" && n.attr("scales")) {
            // opset 7: the scales attribute becomes constant input 1, as the reference's reader does (onnx_registry.rs:1802-1807)
            const onnx::Attribute* a = n.attr("scales");
            onnx::Tensor t;
            t.name = n.name + "/" + (n.outputs.empty() ? std::string() : n.outputs[0]) + "/upsample_scales";
            t.data_type = onnx::DT_FLOAT;
            t.dims = {(int64_t)a->floats.size()};
            t.data.resize(a->floats.size() * 4);
            if (!a->floats.empty()) memcpy(t.data.data(), a->floats.data(), t.data.size());
            const int id = m->value_id(t.name);
            RTB_TRY(upload_constant(m.get(), t, &m->values[(size_t)id]));
            on.n.inputs.resize(2);
            on.n.inputs[1] = t.name;
        }
        for (const std::string& s : on.n.inputs) {
            const int id = m->value_id(s);
            if (id >= 0 && m->values[(size_t)id].kind == V_UNSET)
                return mfail(ctx, RTEN_ERR_INVALID_VALUE, "node '" + n.name + "' (" + n.op_type + ") reads '" + s + "' before it is produced");
            on.in.push_back(id);
        }
        for (const std::string& s : n.outputs) {
            const int id = m->value_id(s);
            if (id >= 0) m->values[(size_t)id].kind = V_TEMP;
            on.out.push_back(id);
        }
        m->nodes.push_back(on);
    }
    for (const onnx::ValueInfo& vi : om.graph.outputs) {
        auto it = m->by_name.find(vi.name);
        if (it == m->by_name.end() || m->values[(size_t)it->second].kind == V_UNSET)
            return mfail(ctx, RTEN_ERR_INVALID_VALUE, "graph output '" + vi.name + "' is never produced");
        m->outputs.push_back(it->second);
    }
    // ---- load-time fusions (src/optimize.rs: the patterns the hot-path models contain)
    auto consumers = [&](int vid) {
        int c = 0;
        for (const OpNode& o : m->nodes)
            for (int i : o.in)
                if (i == vid) c++;
        for (int o : m->outputs)
            if (o == vid) c++;
        return c;
    };
    // SiluFusion (src/optimize/fusions.rs:567-588): Mul(x, Sigmoid(x)), either operand order, becomes Silu(x) when the
    // Sigmoid's output has no other consumer.  Silu rounds once where Mul(x, Sigmoid(x)) rounds twice, so the reference's
    // Model::run computes Silu.  First, because the Sigmoid and the Mul are two consumers of a Conv's output.
    for (size_t i = m->nodes.size(); i-- > 0;) {  // (backwards: erasing node i keeps the indices still to visit)
        OpNode& s = m->nodes[i];
        if (s.n.op_type != "Sigmoid" || s.in.size() != 1 || s.out.size() != 1 || consumers(s.out[0]) != 1) continue;
        size_t j = i + 1;
        for (; j < m->nodes.size(); j++)
            if (std::find(m->nodes[j].in.begin(), m->nodes[j].in.end(), s.out[0]) != m->nodes[j].in.end()) break;
        if (j == m->nodes.size()) continue;
        OpNode& mul = m->nodes[j];
        if (mul.n.op_type != "Mul" || mul.in.size() != 2 || mul.out.size() != 1) continue;
        const int x = s.in[0];
        if (!((mul.in[0] == s.out[0] && mul.in[1] == x) || (mul.in[1] == s.out[0] && mul.in[0] == x))) continue;
        mul.n.op_type = "Silu";
        mul.n.inputs = {s.n.inputs[0]};
        mul.n.attrs.clear();
        mul.in = {x};
        m->nodes.erase(m->nodes.begin() + (long)i);
    }
    for (size_t i = 0; i + 1 < m->nodes.size(); i++) {
        OpNode& a = m->nodes[i];
        if (a.out.size() != 1 || consumers(a.out[0]) != 1) continue;
        // the single consumer
        size_t j = i + 1;
        for (; j < m->nodes.size(); j++)
            if (std::find(m->nodes[j].in.begin(), m->nodes[j].in.end(), a.out[0]) != m->nodes[j].in.end()) break;
        if (j == m->nodes.size()) continue;
        OpNode& b = m->nodes[j];
        if (a.n.op_type == "Conv" && a.activation.kind == RTEN_ACT_NONE && conv_activation(b.n).kind != RTEN_ACT_NONE) {
            a.activation = conv_activation(b.n);  // the activation in the convolution epilogue
            a.out = b.out;
            m->nodes.erase(m->nodes.begin() + (long)j);
        } else if (a.n.op_type == "MatMul" && b.n.op_type == "Add" && a.bias_value < 0 && b.in.size() == 2) {
            // MatMul + Add(constant vector over the last axis) -> FusedMatMul with a row bias (MatMulAddFusion)
            const int other = b.in[0] == a.out[0] ? b.in[1] : b.in[0];
            const ValueSlot& bv = m->values[(size_t)other];
            const ValueSlot& wv = m->values[(size_t)a.in[1]];
            if (bv.kind == V_CONST && bv.t.dtype == RTEN_F32 && bv.t.ndim == 1 && wv.t.ndim >= 2 && wv.kind == V_CONST &&
                bv.t.shape[0] == wv.t.shape[wv.t.ndim - 1]) {
                a.bias_value = other;
                a.out = b.out;
                m->nodes.erase(m->nodes.begin() + (long)j);
            }
        }
    }
    // ---- Concat elision, decided once: which inputs of which channel Concat their producers write in place
    if (!getenv("RTEN_B200_NO_CONCAT_ELISION")) {
        std::map<std::string, std::vector<int64_t>> input_dims;
        for (const onnx::ValueInfo& vi : om.graph.inputs) input_dims[vi.name] = vi.dims;
        auto producer = [&](int vid) {
            for (size_t i = 0; i < m->nodes.size(); i++)
                for (int o : m->nodes[i].out)
                    if (o == vid) return (int)i;
            return -1;
        };
        // channels of a 4-D value as far as the file tells them, else -1
        std::function<int64_t(int, int)> channels = [&](int vid, int depth) -> int64_t {
            if (vid < 0 || depth > 64) return -1;
            const ValueSlot& v = m->values[(size_t)vid];
            if (v.kind == V_INPUT) {
                const std::vector<int64_t>& d = input_dims[v.name];
                return d.size() == 4 && d[1] > 0 ? d[1] : -1;
            }
            const int pi = producer(vid);
            if (pi < 0) return -1;
            const OpNode& p = m->nodes[(size_t)pi];
            const std::string& op = p.n.op_type;
            auto weight = [&]() -> const rten_tensor* {
                if (p.in.size() < 2 || p.in[1] < 0 || m->values[(size_t)p.in[1]].kind != V_CONST) return nullptr;
                const rten_tensor& w = m->values[(size_t)p.in[1]].t;
                return w.ndim == 4 ? &w : nullptr;
            };
            if (op == "Conv") return weight() ? weight()->shape[0] : -1;
            if (op == "ConvTranspose") return weight() ? weight()->shape[1] * p.n.attr_i("group", 1) : -1;
            if (op == "MaxPool" || op == "AveragePool" || op == "Resize" || op == "Upsample" || is_in_place_op(op))
                return channels(p.in[0], depth + 1);
            if (op == "Concat" && p.n.attr_i("axis", 0) == 1) {
                int64_t sum = 0;
                for (int i : p.in) {
                    const int64_t c = channels(i, depth + 1);
                    if (c < 0) return -1;
                    sum += c;
                }
                return sum;
            }
            return -1;
        };
        std::string report;
        for (size_t k = 0; k < m->nodes.size(); k++) {
            OpNode& c = m->nodes[k];
            if (c.n.op_type != "Concat" || c.n.attr_i("axis", 0) != 1 || c.out.size() != 1 || consumers(c.out[0]) < 1) continue;
            std::vector<int64_t> ch;
            for (int i : c.in) ch.push_back(channels(i, 0));
            if (std::find(ch.begin(), ch.end(), (int64_t)-1) != ch.end()) continue;
            std::vector<char> mark(c.in.size(), 0);
            std::string names;
            for (size_t i = 0; i < c.in.size(); i++) {
                const int vid = c.in[i];
                if (m->values[(size_t)vid].kind != V_TEMP) continue;
                if (std::count(c.in.begin(), c.in.end(), vid) != 1) continue;
                if (std::find(m->outputs.begin(), m->outputs.end(), vid) != m->outputs.end()) continue;  // a graph output is copied
                const int pi = producer(vid);
                OpNode& p = m->nodes[(size_t)pi];
                if (!writes_concat_in_place(p.n.op_type) || p.out.size() != 1 || p.cat_node >= 0) continue;
                p.cat_node = (int)k;
                p.cat_slot = (int)i;
                mark[i] = 1;
                names += (names.empty() ? "\"" : ",\"") + m->values[(size_t)vid].name + "\"";
            }
            if (names.empty()) continue;
            c.cat_channels = ch;
            c.cat_in_place = mark;
            report += (report.empty() ? "" : ",") + std::string("{\"output\":\"") + m->values[(size_t)c.out[0]].name +
                      "\",\"copied\":" + std::to_string(std::count(mark.begin(), mark.end(), 0)) + ",\"in_place\":[" + names + "]}";
        }
        // (the summary is the decoded file's JSON object: the plan is appended as one more member)
        const size_t close = m->summary.rfind('}');
        if (close != std::string::npos) m->summary.insert(close, ",\"concat_in_place\":[" + report + "]");
    }
    // ---- prepack constant weights once (Operator::prepack at load, src/graph.rs:488-565)
    for (OpNode& o : m->nodes) {
        const std::string& op = o.n.op_type;
        if ((op == "Conv" || op == "ConvInteger") && o.in.size() >= 2 && m->values[(size_t)o.in[1]].kind == V_CONST &&
            m->values[(size_t)o.in[1]].t.ndim == 4) {
            RTB_TRY(rten_b200_prepack_conv_weight(ctx, &m->values[(size_t)o.in[1]].t, (int)o.n.attr_i("group", 1), &o.packed));
        } else if (op == "ConvTranspose" && o.in.size() >= 2 && m->values[(size_t)o.in[1]].kind == V_CONST &&
                   m->values[(size_t)o.in[1]].t.dtype == RTEN_F32) {
            // (a weight whose attributes the operator would refuse is not prepacked: the run reports the error)
            rten_conv_transpose_params p;
            RTB_TRY(fill_conv_transpose_params(ctx, o.n, &p));
            if (rten_b200_prepack_conv_transpose_weight(ctx, &m->values[(size_t)o.in[1]].t, &p, &o.packed) != RTEN_OK) o.packed = nullptr;
        } else if ((op == "MatMul" || op == "MatMulInteger") && o.in.size() >= 2 && m->values[(size_t)o.in[1]].kind == V_CONST &&
                   m->values[(size_t)o.in[1]].t.ndim == 2) {
            RTB_TRY(rten_b200_prepack_b(ctx, &m->values[(size_t)o.in[1]].t, &o.packed));
        } else if ((op == "GRU" || op == "LSTM") && o.in.size() >= 2 && o.in[1] >= 0 && m->values[(size_t)o.in[1]].kind == V_CONST &&
                   m->values[(size_t)o.in[1]].t.dtype == RTEN_F32 && m->values[(size_t)o.in[1]].t.ndim == 3) {
            // W [dirs, G * H, I] is the input projection's K-major B: prepack it as the [I, dirs * G * H] matrix
            rten_tensor w = m->values[(size_t)o.in[1]].t;
            const int64_t rows = w.shape[0] * w.shape[1], I = w.shape[2];
            w.ndim = 2;
            w.shape[0] = I;
            w.shape[1] = rows;
            w.strides[0] = 1;
            w.strides[1] = I;
            RTB_TRY(rten_b200_prepack_b(ctx, &w, &o.packed));
        }
    }
    RTB_TRY(rten_b200_sync(ctx));
    *out = m.release();
    return RTEN_OK;
}

int32_t rten_b200_model_num_inputs(const rten_model* m) { return m ? (int32_t)m->inputs.size() : 0; }
int32_t rten_b200_model_num_outputs(const rten_model* m) { return m ? (int32_t)m->outputs.size() : 0; }
const char* rten_b200_model_input_name(const rten_model* m, int32_t i) {
    return (m && i >= 0 && i < (int32_t)m->inputs.size()) ? m->values[(size_t)m->inputs[(size_t)i]].name.c_str() : nullptr;
}
const char* rten_b200_model_output_name(const rten_model* m, int32_t i) {
    return (m && i >= 0 && i < (int32_t)m->outputs.size()) ? m->values[(size_t)m->outputs[(size_t)i]].name.c_str() : nullptr;
}
int32_t rten_b200_model_num_nodes(const rten_model* m) { return m ? (int32_t)m->nodes.size() : 0; }
const char* rten_b200_model_node_op(const rten_model* m, int32_t i) {
    return (m && i >= 0 && i < (int32_t)m->nodes.size()) ? m->nodes[(size_t)i].n.op_type.c_str() : nullptr;
}
const char* rten_b200_model_summary(const rten_model* m) { return m ? m->summary.c_str() : nullptr; }

}  // extern "C"

// ------------------------------------------------------------------------------------------
// run
// ------------------------------------------------------------------------------------------
namespace {

struct Runner {
    rten_model* m;
    rten_ctx* ctx;
    std::set<int> keep;  // requested outputs: never released, never overwritten in place
    // A Concat written in place, this run: its buffer (owned by the Concat's output value from the moment the first
    // producer runs) and which inputs are written into it (`on`: the planned ones whose slice starts 16-byte aligned)
    struct CatState {
        bool tried = false, active = false;
        rten_tensor buf{};
        std::vector<char> on;
    };
    std::map<int, CatState> cats;

    ValueSlot& V(int id) { return m->values[(size_t)id]; }
    int root_of(int id) { return V(id).root < 0 ? id : V(id).root; }

    void release_owner(int id) {
        ValueSlot& v = V(id);
        if (v.owned && v.live && v.pending <= 0 && v.views <= 0 && !keep.count(id)) {
            pool_free(ctx, v.t.data);
            v.live = false;
            v.owned = false;
            v.t.data = nullptr;
        }
    }
    void consumed(int id) {
        if (id < 0) return;
        ValueSlot& v = V(id);
        if (v.kind != V_TEMP) return;
        v.pending--;
        if (v.pending > 0) return;
        const int r = root_of(id);
        if (r != id) {
            if (!keep.count(id)) {
                V(r).views--;
                release_owner(r);
            }
        } else {
            release_owner(id);
        }
    }
    void set_owned(int id, const rten_tensor& t) {
        ValueSlot& v = V(id);
        v.t = t;
        v.root = -1;
        v.live = true;
        v.owned = true;
        v.views = 0;
    }
    void set_view(int id, const rten_tensor& t, int src) {
        ValueSlot& v = V(id);
        v.t = t;
        v.live = true;
        v.owned = false;
        const int r = root_of(src);
        if (V(r).kind == V_TEMP && V(r).owned) {
            v.root = r;
            V(r).views++;
        } else {
            v.root = -1;  // view of a constant / graph input: nothing to keep alive
        }
    }

    static bool contiguous(const rten_tensor& t) { return is_contiguous(&t); }

    rten_status make_contiguous(const rten_tensor& src, rten_tensor* dst, bool* allocated) {
        *allocated = false;
        if (contiguous(src)) {
            *dst = src;
            return RTEN_OK;
        }
        rten_tensor c = src;
        set_contiguous(&c);
        void* d = nullptr;
        RTB_TRY(pool_alloc(ctx, (size_t)std::max<int64_t>(numel(&src), 1) * dtype_size(src.dtype), &d));
        c.data = d;
        rten_status st = rten_b200_copy(ctx, &src, &c);
        if (st != RTEN_OK) {
            pool_free(ctx, d);
            return st;
        }
        *dst = c;
        *allocated = true;
        return RTEN_OK;
    }

    rten_status ints_of(int id, std::vector<int64_t>* out) {
        if (id < 0 || !V(id).has_host_ints) return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "shape-like operator input must be a constant");
        *out = V(id).host_ints;
        return RTEN_OK;
    }

    rten_status floats_of(int id, std::vector<float>* out) {
        if (id < 0 || !V(id).has_host_floats) return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "the scales of Resize / Upsample must be a constant");
        *out = V(id).host_floats;
        return RTEN_OK;
    }

    // The target of a Resize (opset 11+: X, roi, scales, sizes; opset 10: X, scales) or Upsample (X, scales) node.  Empty
    // tensors count as missing (src/ops/resize.rs:491-507); roi is ignored, as in the reference.
    rten_status resize_target(const OpNode& o, rten_resize_params* p) {
        RTB_TRY(fill_resize_params(ctx, o.n, p));
        const bool old = o.n.op_type == "Upsample" || o.in.size() == 2;
        const int scales = old ? (o.in.size() > 1 ? o.in[1] : -1) : (o.in.size() > 2 ? o.in[2] : -1);
        const int sizes = (!old && o.in.size() > 3) ? o.in[3] : -1;
        if (scales >= 0 && numel(&V(scales).t) > 0) {
            std::vector<float> f;
            RTB_TRY(floats_of(scales, &f));
            if (V(scales).t.ndim != 1) return mfail(ctx, RTEN_ERR_INVALID_VALUE, "scales must have 1 dims");
            p->n = (int32_t)f.size();
            for (size_t i = 0; i < f.size() && i < 4; i++) p->scales[i] = f[i];
        } else if (sizes >= 0 && numel(&V(sizes).t) > 0) {
            std::vector<int64_t> v;
            RTB_TRY(ints_of(sizes, &v));
            if (V(sizes).t.ndim != 1) return mfail(ctx, RTEN_ERR_INVALID_VALUE, "sizes must have 1 dims");
            p->n = (int32_t)v.size();
            p->use_sizes = 1;
            for (size_t i = 0; i < v.size() && i < 4; i++) p->sizes[i] = v[i];
        } else {
            return mfail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
        }
        return RTEN_OK;
    }

    // Shape [B, C, H, W] a producer of an in-place Concat input will give its output, and whether that output would be
    // channels-last (the operators follow their input's layout).  false: not known here -- the node then runs as usual.
    // A wrong answer cannot corrupt anything: the operator checks the `out` it is given against the shape it computes.
    bool producer_shape(const OpNode& o, int64_t shape[4], bool* channels_last) {
        const rten_tensor& x = V(o.in[0]).t;
        if (x.ndim != 4) return false;
        *channels_last = x.strides[1] == 1 && x.shape[1] > 1;
        const std::string& op = o.n.op_type;
        shape[0] = x.shape[0];
        shape[1] = x.shape[1];
        int64_t p0, p1;
        if (op == "Conv") {
            const rten_tensor& w = V(o.in[1]).t;
            rten_conv_params p;
            if (w.ndim != 4 || fill_conv_params(ctx, o.n, &p) != RTEN_OK) return false;
            shape[1] = w.shape[0];
            for (int a = 0; a < 2; a++)
                if (api::axis_out(ctx, x.shape[2 + a], w.shape[2 + a], p.strides[a], p.auto_pad_same != 0, p.pads[a], p.pads[2 + a],
                                  p.dilations[a], &shape[2 + a], &p0, &p1) != RTEN_OK)
                    return false;
            return true;
        }
        if (op == "ConvTranspose") {  // src/ops/conv_transpose.rs:144-224
            const rten_tensor& w = V(o.in[1]).t;
            rten_conv_transpose_params p;
            if (w.ndim != 4 || fill_conv_transpose_params(ctx, o.n, &p) != RTEN_OK || p.n_strides != 2 || p.n_dilations != 2) return false;
            shape[1] = w.shape[1] * p.groups;
            for (int a = 0; a < 2; a++) {
                const int64_t full = (x.shape[2 + a] - 1) * p.strides[a] + (p.n_output_padding ? p.output_padding[a] : 0) +
                                     (w.shape[2 + a] - 1) * p.dilations[a] + 1;
                shape[2 + a] = p.auto_pad_same ? x.shape[2 + a] * p.strides[a] : full - p.pads[a] - p.pads[2 + a];
            }
            return p.auto_pad_same || p.n_pads == 4;
        }
        if (op == "MaxPool" || op == "AveragePool") {
            PoolAttrs a;
            if (fill_pool_attrs(ctx, o.n, &a) != RTEN_OK) return false;
            for (int i = 0; i < 2; i++)
                if (api::axis_out(ctx, x.shape[2 + i], a.kernel[i], a.strides[i], false, a.pads[i], a.pads[2 + i], 1, &shape[2 + i], &p0, &p1) != RTEN_OK)
                    return false;
            return true;
        }
        if (op == "Resize" || op == "Upsample") {  // calc_output_size (src/ops/resize.rs:287-298)
            rten_resize_params p;
            if (resize_target(o, &p) != RTEN_OK || p.n != 4) return false;
            for (int i = 0; i < 4; i++) {
                const volatile float prod = (float)x.shape[i] * p.scales[i];
                const int64_t d = p.use_sizes ? p.sizes[i] : (int64_t)floorf(prod);
                if (i < 2 && d != x.shape[i]) return false;
                shape[i] = d;
            }
            return true;
        }
        return false;
    }

    // `out` for a node whose output is planned to be written into a Concat's buffer: the strided view of its channel
    // slice, allocating the buffer when this is the first such producer to run.  false: the node allocates as usual.
    bool concat_slice(const OpNode& o, rten_tensor* slice) {
        OpNode& c = m->nodes[(size_t)o.cat_node];
        CatState& cs = cats[o.cat_node];
        int64_t shape[4];
        bool cl = false;
        if (!producer_shape(o, shape, &cl)) return false;
        const size_t n = c.cat_channels.size();
        if (!cs.tried) {
            cs.tried = true;
            int64_t total = 0;
            for (int64_t ch : c.cat_channels) total += ch;
            rten_tensor b{};
            b.dtype = RTEN_F32;
            b.ndim = 4;
            b.device = ctx->device;
            b.shape[0] = shape[0], b.shape[1] = total, b.shape[2] = shape[2], b.shape[3] = shape[3];
            b.strides[0] = total * shape[2] * shape[3];
            b.strides[1] = cl ? 1 : shape[2] * shape[3];
            b.strides[2] = cl ? shape[3] * total : shape[3];
            b.strides[3] = cl ? total : 1;
            cs.on.assign(n, 0);
            int64_t start = 0;
            bool any = false;
            for (size_t i = 0; i < n; i++) {
                cs.on[i] = c.cat_in_place[i] && (start * b.strides[1]) % 4 == 0;  // the slice starts 16-byte aligned
                any = any || cs.on[i];
                start += c.cat_channels[i];
            }
            if (!any || numel(&b) == 0) return false;
            if (pool_alloc(ctx, (size_t)numel(&b) * 4, &b.data) != RTEN_OK) return false;
            cs.buf = b;
            cs.active = true;
            set_owned(c.out[0], b);
        }
        if (!cs.active || !cs.on[(size_t)o.cat_slot]) return false;
        const rten_tensor& b = cs.buf;
        if (shape[0] != b.shape[0] || shape[1] != c.cat_channels[(size_t)o.cat_slot] || shape[2] != b.shape[2] || shape[3] != b.shape[3])
            return false;  // (the Concat node will report the mismatch)
        int64_t start = 0;
        for (int i = 0; i < o.cat_slot; i++) start += c.cat_channels[(size_t)i];
        *slice = b;
        slice->shape[1] = shape[1];
        slice->data = (float*)b.data + start * b.strides[1];
        return true;
    }

    rten_status run_view(OpNode& o) {
        const std::string& op = o.n.op_type;
        const rten_tensor& x = V(o.in[0]).t;
        rten_tensor y = x;
        int src = o.in[0];
        if (op == "Transpose") {
            std::vector<int64_t> perm = o.n.attr_ints("perm");
            if (perm.empty())
                for (int i = x.ndim - 1; i >= 0; i--) perm.push_back(i);
            if ((int)perm.size() != x.ndim) return mfail(ctx, RTEN_ERR_INVALID_VALUE, "Transpose: perm has the wrong length");
            for (int i = 0; i < x.ndim; i++) {
                const int64_t a = perm[(size_t)i];
                if (a < 0 || a >= x.ndim) return mfail(ctx, RTEN_ERR_INVALID_VALUE, "Transpose: perm entry out of range");
                y.shape[i] = x.shape[a];
                y.strides[i] = x.strides[a];
            }
            set_view(o.out[0], y, src);
            return RTEN_OK;
        }
        if (op == "Identity") {
            set_view(o.out[0], y, src);
            return RTEN_OK;
        }
        // the remaining view operators re-shape: the data must be contiguous first
        rten_tensor c;
        bool alloc = false;
        RTB_TRY(make_contiguous(x, &c, &alloc));
        std::vector<int64_t> shape;
        const int64_t total = numel(&c);
        if (op == "Reshape") {
            std::vector<int64_t> want;
            RTB_TRY(ints_of(o.in.size() > 1 ? o.in[1] : -1, &want));
            int64_t known = 1;
            int infer = -1;
            for (size_t i = 0; i < want.size(); i++) {
                int64_t d = want[i];
                if (d == 0 && !o.n.attr_i("allowzero", 0)) d = (int)i < c.ndim ? c.shape[i] : 0;
                if (d == -1) {
                    if (infer >= 0) return mfail(ctx, RTEN_ERR_INVALID_VALUE, "Multiple dimensions in new shape set to -1");
                    infer = (int)i;
                    d = 1;
                }
                shape.push_back(d);
                known *= d;
            }
            if (infer >= 0) {
                if (known == 0 || total % known) return mfail(ctx, RTEN_ERR_INVALID_VALUE, "Input length must be a multiple of specified dimensions");
                shape[(size_t)infer] = total / known;
            }
        } else if (op == "Flatten") {
            int64_t axis = o.n.attr_i("axis", 1);
            if (axis < 0) axis += c.ndim;
            int64_t a = 1, b = 1;
            for (int i = 0; i < c.ndim; i++) (i < axis ? a : b) *= c.shape[i];
            shape = {a, b};
        } else {  // Squeeze / Unsqueeze: axes attribute (opset < 13) or second input
            std::vector<int64_t> axes = o.n.attr_ints("axes");
            if (axes.empty() && o.in.size() > 1 && o.in[1] >= 0) RTB_TRY(ints_of(o.in[1], &axes));
            if (op == "Squeeze") {
                for (int i = 0; i < c.ndim; i++) {
                    bool drop = axes.empty() ? c.shape[i] == 1 : false;
                    for (int64_t a : axes)
                        if ((a < 0 ? a + c.ndim : a) == i) drop = true;
                    if (!drop) shape.push_back(c.shape[i]);
                }
            } else {
                const int nd = c.ndim + (int)axes.size();
                std::vector<bool> ins((size_t)nd, false);
                for (int64_t a : axes) {
                    const int64_t p = a < 0 ? a + nd : a;
                    if (p < 0 || p >= nd) return mfail(ctx, RTEN_ERR_INVALID_VALUE, "Axes must be in range [-r, r-1]");
                    ins[(size_t)p] = true;
                }
                int k = 0;
                for (int i = 0; i < nd; i++) shape.push_back(ins[(size_t)i] ? 1 : c.shape[k++]);
            }
        }
        int64_t prod = 1;
        for (int64_t d : shape) prod *= d;
        if (prod != total) return mfail(ctx, RTEN_ERR_INVALID_VALUE, "New shape must have same total elements as current shape");
        if ((int)shape.size() > RTEN_MAX_DIMS) return mfail(ctx, RTEN_ERR_INVALID_VALUE, "tensor rank out of range");
        y = c;
        y.ndim = (int)shape.size();
        for (int i = 0; i < y.ndim; i++) y.shape[i] = shape[(size_t)i];
        set_contiguous(&y);
        if (alloc)
            set_owned(o.out[0], y);
        else
            set_view(o.out[0], y, src);
        return RTEN_OK;
    }

    rten_status run_node(OpNode& o) {
        const std::string& op = o.n.op_type;
        auto T = [&](size_t i) -> const rten_tensor* { return (i < o.in.size() && o.in[i] >= 0) ? &V(o.in[i]).t : nullptr; };
        if (!T(0)) return mfail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
        if (is_view_op(op)) return run_view(o);
        rten_tensor y;
        memset(&y, 0, sizeof(y));
        rten_status st = RTEN_OK;
        // in place when the executor holds the last reference to input 0 (src/graph.rs:973-1049)
        bool in_place = false;
        if (is_in_place_op(op)) {
            ValueSlot& x = V(o.in[0]);
            in_place = x.kind == V_TEMP && x.owned && x.root < 0 && x.pending == 1 && x.views == 0 && !keep.count(o.in[0]) && contiguous(x.t);
            if (in_place) y = x.t;
        }
        const bool into_concat = o.cat_node >= 0 && concat_slice(o, &y);
        if (op == "Conv" || op == "ConvInteger") {
            rten_conv_params p;
            RTB_TRY(fill_conv_params(ctx, o.n, &p));
            if (op == "Conv")
                st = rten_b200_conv2d_act(ctx, T(0), T(1), o.packed, T(2), &p, nullptr, &o.activation, &y);
            else
                st = rten_b200_conv_integer(ctx, T(0), T(1), o.packed, T(2), T(3), nullptr, &p, &y);
        } else if (op == "ConvTranspose") {
            rten_conv_transpose_params p;
            RTB_TRY(fill_conv_transpose_params(ctx, o.n, &p));
            st = rten_b200_conv_transpose(ctx, T(0), T(1), o.packed, T(2), &p, &y);
        } else if (op == "Relu") {
            st = rten_b200_relu(ctx, T(0), &y);
        } else if (op == "Clip") {
            st = rten_b200_clip(ctx, T(0), T(1), T(2), &y);
        } else if (op == "Sigmoid") {
            st = rten_b200_sigmoid(ctx, T(0), &y);
        } else if (op == "Silu") {
            st = rten_b200_silu(ctx, T(0), &y);
        } else if (op == "HardSigmoid") {
            st = rten_b200_hard_sigmoid(ctx, T(0), hard_sigmoid_alpha(o.n), hard_sigmoid_beta(o.n), &y);
        } else if (op == "HardSwish") {
            st = rten_b200_hard_swish(ctx, T(0), &y);
        } else if (op == "Gelu") {
            const onnx::Attribute* a = o.n.attr("approximate");
            st = rten_b200_gelu(ctx, T(0), (a && a->s == "tanh") ? 1 : 0, &y);
        } else if (op == "Erf") {
            st = rten_b200_erf(ctx, T(0), &y);
        } else if (op == "Softmax") {
            st = rten_b200_softmax(ctx, T(0), nullptr, (int)o.n.attr_i("axis", -1), 0, &y);
        } else if (op == "MaxPool" || op == "AveragePool") {
            PoolAttrs a;
            RTB_TRY(fill_pool_attrs(ctx, o.n, &a));
            if (op == "MaxPool")
                st = rten_b200_max_pool(ctx, T(0), a.kernel, a.pads, a.strides, &y);
            else
                st = rten_b200_average_pool(ctx, T(0), a.kernel, a.pads, a.strides, (int)o.n.attr_i("count_include_pad", 0), &y);
        } else if (op == "Resize" || op == "Upsample") {
            rten_resize_params p;
            RTB_TRY(resize_target(o, &p));
            st = rten_b200_resize(ctx, T(0), &p, &y);
        } else if (op == "Concat") {
            std::vector<const rten_tensor*> ins;
            for (size_t i = 0; i < o.in.size(); i++)
                if (T(i)) ins.push_back(T(i));
            auto cs = cats.find((int)(&o - m->nodes.data()));
            if (cs != cats.end() && cs->second.active) {
                // the buffer is the output value already; inputs that are their slice of it are skipped by the operator
                rten_tensor b = cs->second.buf;
                return rten_b200_concat(ctx, ins.data(), (int)ins.size(), (int)o.n.attr_i("axis", 0), &b);
            }
            st = rten_b200_concat(ctx, ins.data(), (int)ins.size(), (int)o.n.attr_i("axis", 0), &y);
        } else if (op == "GlobalAveragePool" || op == "ReduceMean") {
            const rten_tensor* x = T(0);
            bool keepdims = true;
            if (op == "ReduceMean") {
                std::vector<int64_t> axes = o.n.attr_ints("axes");
                if (axes.empty() && o.in.size() > 1 && o.in[1] >= 0) RTB_TRY(ints_of(o.in[1], &axes));
                keepdims = o.n.attr_i("keepdims", 1) != 0;
                bool spatial = x->ndim == 4 && axes.size() == 2;
                for (int64_t a : axes) {
                    const int64_t p = a < 0 ? a + x->ndim : a;
                    if (p != 2 && p != 3) spatial = false;
                }
                if (!spatial) return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "ReduceMean: only the spatial axes of an NCHW tensor are supported");
            }
            st = rten_b200_global_average_pool(ctx, x, &y);
            if (st == RTEN_OK && !keepdims) {
                y.ndim = 2;
                set_contiguous(&y);
            }
        } else if (op == "Gemm") {
            st = rten_b200_gemm(ctx, T(0), T(1), T(2), o.n.attr_f("alpha", 1.0f), o.n.attr_f("beta", 1.0f), (int)o.n.attr_i("transA", 0),
                                (int)o.n.attr_i("transB", 0), &y);
        } else if (op == "MatMul") {
            const rten_tensor* bias = o.bias_value >= 0 ? &V(o.bias_value).t : nullptr;
            st = rten_b200_matmul(ctx, T(0), T(1), o.packed, bias, 1.0f, &y);
        } else if (op == "MatMulInteger") {
            st = rten_b200_matmul_integer(ctx, T(0), T(1), o.packed, T(2), T(3), nullptr, &y);
        } else if (op == "MatMulNBits") {
            // accuracy_level only sets a minimum: every level computes in f32 (src/ops/matmul/contrib.rs:104-109)
            if (o.in.size() > 3) return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "zero_points, g_idx and bias inputs are unsupported");
            if (!T(1) || !T(2)) return mfail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
            st = rten_b200_matmul_nbits(ctx, T(0), T(1), T(2), 4, (int)o.n.attr_i("block_size", 0), &y);
        } else if (op == "Add") {
            if (!T(1)) return mfail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
            st = rten_b200_add(ctx, T(0), T(1), &y);
        } else if (op == "Mul") {
            if (!T(1)) return mfail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
            st = rten_b200_mul(ctx, T(0), T(1), &y);
        } else if (op == "LayerNormalization") {
            st = rten_b200_layer_norm(ctx, T(0), T(1), T(2), (int)o.n.attr_i("axis", -1), o.n.attr_f("epsilon", 1e-5f), &y);
        } else if (op == "RMSNormalization" || op == "SimplifiedLayerNormalization") {
            if (!T(1)) return mfail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
            st = rten_b200_rms_norm(ctx, T(0), T(1), (int)o.n.attr_i("axis", -1), o.n.attr_f("epsilon", 1e-5f), &y);
        } else if (op == "SkipLayerNormalization" || op == "SkipSimplifiedLayerNormalization") {
            // inputs: x, skip, gamma, beta, bias (SkipLayerNormalization); x, skip, gamma, bias (the simplified one)
            const bool rms = op == "SkipSimplifiedLayerNormalization";
            const bool want_sum = o.out.size() > 3 && o.out[3] >= 0;
            rten_tensor s;
            memset(&s, 0, sizeof(s));
            st = rten_b200_skip_layer_norm(ctx, T(0), T(1), T(2), rms ? nullptr : T(3), rms ? T(3) : T(4), o.n.attr_f("epsilon", 0.0f),
                                           rms ? 1 : 0, &y, want_sum ? &s : nullptr);
            if (st == RTEN_OK && want_sum) set_owned(o.out[3], s);
        } else if (op == "Gather") {
            if (o.n.attr_i("axis", 0) != 0 || T(0)->ndim != 2)
                return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "Gather: only axis 0 of a 2-D table is supported");
            st = rten_b200_gather_rows(ctx, T(0), T(1), &y);
        } else if (op == "DynamicQuantizeLinear") {
            rten_tensor s, z;
            memset(&s, 0, sizeof(s));
            memset(&z, 0, sizeof(z));
            st = rten_b200_dynamic_quantize_linear(ctx, T(0), &y, &s, &z, nullptr);
            if (st == RTEN_OK) {
                if (o.out.size() > 1 && o.out[1] >= 0) set_owned(o.out[1], s); else pool_free(ctx, s.data);
                if (o.out.size() > 2 && o.out[2] >= 0) set_owned(o.out[2], z); else pool_free(ctx, z.data);
            }
        } else if (op == "Cast") {
            const int64_t to = o.n.attr_i("to", 0);
            const rten_tensor* x = T(0);
            if (to == onnx::DT_FLOAT && x->dtype == RTEN_I32) {
                rten_tensor c;
                bool alloc = false;
                RTB_TRY(make_contiguous(*x, &c, &alloc));
                y = c;
                y.dtype = RTEN_F32;
                void* d = nullptr;
                st = pool_alloc(ctx, (size_t)std::max<int64_t>(numel(&c), 1) * 4, &d);
                if (st == RTEN_OK) {
                    y.data = d;
                    const long long n = numel(&c);
                    st = launch_cast_scale(ctx, (const int*)c.data, (float*)d, n, 1, m->one, 1);  // f32(x) * 1.0f: exact
                }
                if (alloc) pool_free(ctx, c.data);
            } else if ((to == onnx::DT_FLOAT && x->dtype == RTEN_F32) || ((to == onnx::DT_INT32 || to == onnx::DT_INT64) && x->dtype == RTEN_I32)) {
                set_view(o.out[0], *x, o.in[0]);
                return RTEN_OK;
            } else {
                return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "Cast: only int32 -> float is supported");
            }
        } else if (op == "Attention") {
            rten_attention_params p;
            memset(&p, 0, sizeof(p));
            p.is_causal = (int32_t)o.n.attr_i("is_causal", 0);
            p.q_num_heads = (int32_t)o.n.attr_i("q_num_heads", 0);
            p.kv_num_heads = (int32_t)o.n.attr_i("kv_num_heads", 0);
            p.scale = o.n.attr_f("scale", 0.0f);
            p.softcap = o.n.attr_f("softcap", 0.0f);
            if (T(4) || T(5)) return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "Attention: past_key / past_value inputs are not supported by the executor");
            st = rten_b200_attention(ctx, T(0), T(1), T(2), T(3), T(6), &p, nullptr, nullptr, &y);
        } else if (op == "RotaryEmbedding") {
            if (!T(1) || !T(2)) return mfail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
            st = rten_b200_rotary_embedding(ctx, T(0), T(1), T(2), T(3), (int)o.n.attr_i("interleaved", 0), (int)o.n.attr_i("num_heads", 0),
                                            (int)o.n.attr_i("rotary_embedding_dim", 0), &y);
        } else if (op == "GroupQueryAttention") {
            if (T(11)) return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "head_sink is not supported");
            if (o.n.attr_i("smooth_softmax", 0)) return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "smooth_softmax is not supported");
            rten_gqa_params p;
            memset(&p, 0, sizeof(p));
            p.num_heads = (int32_t)o.n.attr_i("num_heads", 0);
            p.kv_num_heads = (int32_t)o.n.attr_i("kv_num_heads", 0);
            p.scale = o.n.attr_f("scale", 0.0f);
            p.do_rotary = (int32_t)o.n.attr_i("do_rotary", 0);
            p.rotary_interleaved = (int32_t)o.n.attr_i("rotary_interleaved", 0);
            p.local_window_size = (int32_t)o.n.attr_i("local_window_size", -1);
            p.softcap = o.n.attr_f("softcap", 0.0f);
            if (!T(5) || !T(6)) return mfail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
            rten_tensor pk, pv;
            memset(&pk, 0, sizeof(pk));
            memset(&pv, 0, sizeof(pv));
            st = rten_b200_group_query_attention(ctx, T(0), T(1), T(2), T(3), T(4), T(5), T(6), T(7), T(8), T(9), T(10), &p, &y, &pk, &pv);
            if (st == RTEN_OK) {
                if (o.out.size() > 1 && o.out[1] >= 0) set_owned(o.out[1], pk); else pool_free(ctx, pk.data);
                if (o.out.size() > 2 && o.out[2] >= 0) set_owned(o.out[2], pv); else pool_free(ctx, pv.data);
            }
        } else if (op == "MultiHeadAttention") {
            rten_mha_params p;
            memset(&p, 0, sizeof(p));
            p.num_heads = (int32_t)o.n.attr_i("num_heads", 0);
            p.scale = o.n.attr_f("scale", 0.0f);
            p.mask_filter_value = o.n.attr_f("mask_filter_value", -10000.0f);
            p.unidirectional = (int32_t)o.n.attr_i("unidirectional", 0);
            const bool want_k = o.out.size() > 1 && o.out[1] >= 0, want_v = o.out.size() > 2 && o.out[2] >= 0;
            rten_tensor pk, pv;
            memset(&pk, 0, sizeof(pk));
            memset(&pv, 0, sizeof(pv));
            st = rten_b200_multi_head_attention(ctx, T(0), T(1), T(2), T(3), T(4), T(5), T(6), T(7), nullptr, nullptr, &p, &y,
                                                want_k ? &pk : nullptr, want_v ? &pv : nullptr);
            if (st == RTEN_OK) {
                if (want_k) set_owned(o.out[1], pk);
                if (want_v) set_owned(o.out[2], pv);
            }
        } else if (op == "GRU" || op == "LSTM") {
            const bool gru = op == "GRU";
            rten_rnn_params p;
            memset(&p, 0, sizeof(p));
            p.direction = rnn_direction(o.n);
            p.hidden_size = (int32_t)o.n.attr_i("hidden_size", 0);
            p.linear_before_reset = (int32_t)o.n.attr_i("linear_before_reset", 0);
            auto want = [&](size_t i) { return o.out.size() > i && o.out[i] >= 0; };
            rten_tensor ys[3];
            memset(ys, 0, sizeof(ys));
            if (gru)
                st = rten_b200_gru(ctx, T(0), T(1), o.packed, T(2), T(3), T(4), T(5), &p, want(0) ? &ys[0] : nullptr,
                                   want(1) ? &ys[1] : nullptr);
            else
                st = rten_b200_lstm(ctx, T(0), T(1), o.packed, T(2), T(3), T(4), T(5), T(6), nullptr, &p,
                                    want(0) ? &ys[0] : nullptr, want(1) ? &ys[1] : nullptr, want(2) ? &ys[2] : nullptr);
            RTB_TRY(st);
            for (size_t i = 0; i < 3; i++)
                if (want(i) && (i < 2 || !gru)) set_owned(o.out[i], ys[i]);
            return RTEN_OK;
        } else {
            return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "unsupported operator " + op);
        }
        RTB_TRY(st);
        if (in_place) {
            // the input's buffer now belongs to the output value
            ValueSlot& x = V(o.in[0]);
            x.owned = false;
            x.live = false;
        }
        if (into_concat)
            set_view(o.out[0], y, m->nodes[(size_t)o.cat_node].out[0]);
        else
            set_owned(o.out[0], y);
        return RTEN_OK;
    }
};

}  // namespace

extern "C" rten_status rten_b200_model_run(rten_model* m, int32_t n_inputs, const char* const* input_names, const rten_tensor* inputs,
                                           int32_t n_outputs, const char* const* output_names, rten_tensor* outputs) {
    if (!m || (n_inputs && (!input_names || !inputs)) || n_outputs < 1 || !output_names || !outputs) return RTEN_ERR_INVALID_VALUE;
    rten_ctx* ctx = m->ctx;
    cudaSetDevice(ctx->device);
    Runner r{m, ctx, {}, {}};
    // reset run state
    for (ValueSlot& v : m->values) {
        if (v.kind == V_TEMP || v.kind == V_INPUT) {
            v.live = false;
            v.owned = false;
            v.root = -1;
            v.views = 0;
            v.pending = 0;
            if (v.kind == V_TEMP) v.t.data = nullptr;
        }
    }
    std::vector<void*> staged;  // device copies of host inputs
    auto cleanup = [&](rten_status st) {
        for (ValueSlot& v : m->values)
            if (v.kind == V_TEMP && v.owned && v.live && (st != RTEN_OK || !r.keep.count((int)(&v - m->values.data())))) {
                pool_free(ctx, v.t.data);
                v.live = false;
                v.owned = false;
            }
        for (void* p : staged) pool_free(ctx, p);
        return st;
    };
    for (int32_t i = 0; i < n_inputs; i++) {
        auto it = m->by_name.find(input_names[i] ? input_names[i] : "");
        if (it == m->by_name.end() || m->values[(size_t)it->second].kind != V_INPUT)
            return mfail(ctx, RTEN_ERR_INVALID_VALUE, std::string("unknown model input '") + (input_names[i] ? input_names[i] : "") + "'");
        ValueSlot& v = m->values[(size_t)it->second];
        v.t = inputs[i];
        if (inputs[i].device < 0) {  // host tensor: staged through HBM for the duration of the run
            rten_tensor d = inputs[i];
            set_contiguous(&d);
            void* p = nullptr;
            rten_status st = pool_alloc(ctx, (size_t)std::max<int64_t>(numel(&d), 1) * dtype_size(d.dtype), &p);
            if (st != RTEN_OK) return cleanup(st);
            staged.push_back(p);
            d.data = p;
            d.device = ctx->device;
            st = rten_b200_copy(ctx, &inputs[i], &d);
            if (st != RTEN_OK) return cleanup(st);
            v.t = d;
        }
        v.live = true;
    }
    for (int id : m->inputs)
        if (!m->values[(size_t)id].live) return cleanup(mfail(ctx, RTEN_ERR_MISSING_INPUTS, "model input '" + m->values[(size_t)id].name + "' was not provided"));
    std::vector<int> want;
    for (int32_t i = 0; i < n_outputs; i++) {
        auto it = m->by_name.find(output_names[i] ? output_names[i] : "");
        if (it == m->by_name.end()) return cleanup(mfail(ctx, RTEN_ERR_INVALID_VALUE, std::string("unknown model output '") + (output_names[i] ? output_names[i] : "") + "'"));
        want.push_back(it->second);
        r.keep.insert(it->second);
    }
    // consumer counts (the plan is the whole node list: pruning to the requested outputs is not needed for these models)
    for (OpNode& o : m->nodes) {
        for (int i : o.in)
            if (i >= 0) m->values[(size_t)i].pending++;
        if (o.bias_value >= 0) m->values[(size_t)o.bias_value].pending++;
    }
    for (OpNode& o : m->nodes) {
        rten_status st = r.run_node(o);
        if (st != RTEN_OK) return cleanup(st);
        std::set<int> seen;
        for (int i : o.in) r.consumed(i);
        (void)seen;
    }
    // hand the requested outputs over: owned buffers move to the caller; views / constants / inputs are copied
    for (int32_t i = 0; i < n_outputs; i++) {
        ValueSlot& v = m->values[(size_t)want[(size_t)i]];
        if (!v.live && v.kind != V_CONST) return cleanup(mfail(ctx, RTEN_ERR_INVALID_VALUE, "requested output '" + v.name + "' was not computed"));
        const bool movable = v.kind == V_TEMP && v.owned && v.root < 0 && v.views == 0 && is_contiguous(&v.t);
        bool dup = false;
        for (int32_t k = 0; k < i; k++) dup = dup || want[(size_t)k] == want[(size_t)i];
        if (movable && !dup) {
            outputs[i] = v.t;
            v.owned = false;
            v.live = false;
        } else {
            rten_tensor c = v.t;
            set_contiguous(&c);
            void* p = nullptr;
            rten_status st = pool_alloc(ctx, (size_t)std::max<int64_t>(numel(&c), 1) * dtype_size(c.dtype), &p);
            if (st != RTEN_OK) return cleanup(st);
            c.data = p;
            st = rten_b200_copy(ctx, &v.t, &c);
            if (st != RTEN_OK) {
                pool_free(ctx, p);
                return cleanup(st);
            }
            outputs[i] = c;
        }
    }
    r.keep.clear();
    return cleanup(RTEN_OK);
}
