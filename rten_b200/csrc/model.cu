// Minimal graph executor behind the C ABI (include/rten_b200.h: rten_b200_model_*): what RTen's `Model::load` +
// `Graph::run_plan` do around the operators of this library (src/model.rs, src/graph.rs:880-1286), restated for the
// hot-path operator set:
//   load : build_graph (ONNX bytes -> nodes + initialisers, onnx_reader.cu; int64 tensors become i32 like rten's loader
//          does; constants uploaded to HBM once) -> the fusions of src/optimize.rs the models need, in this order:
//          fuse_silu, fuse_group_norm, fold_batch_norm, fuse_into_producers -> plan_concat_elision -> prepack_weights
//          (src/graph.rs:488-565).  fold_batch_norm is this executor's own: a BatchNormalization that is the only reader of
//          an f32 Conv / ConvTranspose with constant weights goes into those weights and bias, as export tools fold it.
//          The folded convolution rounds each weight product once more than the reference's Conv then
//          BatchNormalization, so its output is held to the f32 convolution tolerance, not bit for bit -- depthwise
//          layers included, whose unfolded kernel is bit-identical to the reference.
//   run  : the nodes in topological (file) order, one C-ABI operator call each; temporaries are reference counted and
//          returned to the context pool after their last consumer (src/graph.rs:1100-1180); an operator that can run in
//          place does so when the executor holds the last reference to its input (src/graph.rs:973-1049); shape-only
//          operators (Reshape, Flatten, Squeeze, Unsqueeze, Transpose, Identity) and Slice / Split are views -- no kernel,
//          no copy.
//          Shape-like values are computed on the host (Runner::set_host): Shape, a Gather of a host-known vector with
//          host-known indices, an integer Cast, the order-keeping views of such values, and Add / Sub / Mul / Div, the
//          comparisons, Where, Concat and Slice of host-known inputs, i32 Range and integer ConstantOfShape launch nothing, so a Reshape
//          target or the total_sequence_length of onnxruntime-genai's attention-mask subgraph is known without a copy
//          back; an operator that takes one as a tensor gets a host tensor (GroupQueryAttention reads it in place).
//          A Concat over the channels of NCHW tensors is written in place by its producers where the load found that
//          possible (plan_concat_elision): the first such producer to run allocates the Concat's buffer and every one of
//          them gets a strided view of its channel slice as `out`, so the Concat node copies only the other inputs --
//          nothing when there are none.  RTEN_B200_NO_CONCAT_ELISION=1 (read at load) turns that off for comparisons.
// Operators: the table OPS, one row per (domain, op_type) the executor accepts.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <set>
#include <string>
#include <string_view>
#include <vector>

#include "api_shared.h"
#include "api_util.h"
#include "masks.h"
#include "onnx_reader.h"
#include "rowops.h"

using namespace rtb;

namespace {

enum ValueKind { V_UNSET = 0, V_CONST, V_INPUT, V_TEMP };

struct ValueSlot {
    std::string name;
    ValueKind kind = V_UNSET;
    rten_tensor t{};
    // shape-like value known on the host: usable by Reshape / axes inputs.  A constant (int64 in the file), or a run-time
    // value computed on the host from shapes (Shape, Gather, Cast and the views of such values), whose tensor is then a
    // host tensor over host_i32 for the rest of the run.
    bool has_host_ints = false;
    std::vector<int64_t> host_ints;
    std::vector<int32_t> host_i32;
    bool has_host_floats = false;     // small f32 constant: usable as the scales of Resize / Upsample
    std::vector<float> host_floats;
    // run state
    int root = -1;        // value that owns the allocation (self for owners)
    int pending = 0;      // consumers still to run
    int views = 0;        // live views of this owner
    bool live = false;
    bool owned = false;   // allocation belongs to the executor (pool)
    // a graph input the caller made writable (rten_b200_model_run_ex): its buffer holds `capacity` positions along
    // `grow_axis`; input_index is its index in the call's inputs.  On any value: the writable input whose buffer it is a
    // view of (an in-place present cache), else -1.
    bool writable = false;
    int grow_axis = -1;
    int64_t capacity = 0;
    int input_index = -1, alias_of = -1;
};

struct OpNode;
struct Runner;

enum OpDomain : uint8_t { ONNX = 1, MS = 2 };  // "" or "ai.onnx"; "com.microsoft"
enum OpFlag : uint8_t { VIEW = 1, IN_PLACE = 2, RESHAPE = 4 };

// What the executor knows about one operator: a row of OPS
struct OpDef {
    const char* name;
    uint8_t domains;    // OpDomain bits; none for an operator only a fusion makes
    uint8_t flags;      // VIEW: no kernel (Runner::run_view), RESHAPE: of contiguous data; IN_PLACE: may overwrite input 0
    uint32_t required;  // bit i: input i must be present when the node runs
    rten_status (*run)(Runner& r, OpNode& o, rten_tensor* y);  // one C-ABI call; outputs > 0 through Runner::set_output
    rten_status (*load)(rten_model* m, onnx::Node& n) = nullptr;  // load-time checks; legacy attributes become inputs
    rten_status (*prepack)(rten_ctx* ctx, OpNode& o, const rten_tensor& w) = nullptr;  // of the constant input 1, at load
    // Output 0's shape for the NCHW input `x` (`shape` preset to x's): the operator can write a Concat's channel slice
    // in place.  The convolutions' store paths take the output's pixel and channel strides, ConvTranspose's stride
    // phases are such views already, the pooling and Resize kernels index with the output strides.  Not the elementwise
    // operators: they reach a strided `out` through a temporary and a copy, which costs what the Concat copy costs; nor
    // a nested Concat, whose buffer would have to exist before its own.
    bool (*shape)(Runner& r, const OpNode& o, const rten_tensor& x, int64_t shape[4]) = nullptr;
    rten_activation_kind act = RTEN_ACT_NONE;  // the Conv epilogue activation this operator fuses into
};

struct OpNode {
    onnx::Node n;
    const OpDef* def = nullptr;
    std::vector<int> in, out;  // value ids (-1 = absent optional input)
    rten_packed* packed = nullptr;
    rten_activation activation = {RTEN_ACT_NONE, 0.0f, 0.0f};  // fused activation of a Conv or GroupNorm
    int bias_value = -1;       // fused Add(bias) of a MatMul (fuse_into_producers)
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
rten_status upload_constant(rten_model* m, const onnx::Tensor& t) {
    rten_ctx* ctx = m->ctx;
    ValueSlot* v = &m->values[(size_t)m->value_id(t.name)];
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

// A float attribute of an older opset as constant input `slot`, as the reference's reader does: Clip's min / max
// (opset < 11, src/op_registry/onnx_registry.rs:887-898) as scalars, Upsample's scales (opset 7, :1802-1807) as a list
rten_status attr_to_input(rten_model* m, onnx::Node& n, const char* attr, size_t slot, const char* suffix, bool scalar) {
    const onnx::Attribute* a = n.attr(attr);
    if (!a) return RTEN_OK;
    const std::vector<float> v = scalar ? std::vector<float>{a->f} : a->floats;
    onnx::Tensor t;
    t.name = n.name + "/" + (n.outputs.empty() ? std::string() : n.outputs[0]) + "/" + suffix;
    t.data_type = onnx::DT_FLOAT;
    if (!scalar) t.dims = {(int64_t)v.size()};
    t.data.resize(v.size() * 4);
    if (!v.empty()) memcpy(t.data.data(), v.data(), t.data.size());
    RTB_TRY(upload_constant(m, t));
    if (n.inputs.size() <= slot) n.inputs.resize(slot + 1);
    n.inputs[slot] = t.name;
    return RTEN_OK;
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
rten_status check_rnn_attrs(rten_ctx* ctx, const onnx::Node& n, bool gru) {
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

rten_rnn_params rnn_params(const onnx::Node& n) {
    rten_rnn_params p;
    memset(&p, 0, sizeof(p));
    p.direction = rnn_direction(n);
    p.hidden_size = (int32_t)n.attr_i("hidden_size", 0);
    p.linear_before_reset = (int32_t)n.attr_i("linear_before_reset", 0);
    return p;
}

// HardSigmoid's attributes with the reference's defaults (src/op_registry/onnx_registry.rs:1228-1232)
float hard_sigmoid_alpha(const onnx::Node& n) { return n.attr_f("alpha", 0.2f); }
float hard_sigmoid_beta(const onnx::Node& n) { return n.attr_f("beta", 0.5f); }

// Resize / Upsample attributes as the reference reads them (src/op_registry/onnx_registry.rs:1721-1778, 1789-1810):
// antialias, exclude_outside, extrapolation_value, keep_aspect_ratio_policy and cubic_coeff_a must have their defaults;
// `cubic` falls back to linear; defaults nearest, round_prefer_floor, half_pixel.  Upsample is always asymmetric + floor
// (src/ops/resize.rs:629-642).
rten_status fill_resize_params(rten_ctx* ctx, const onnx::Node& n, bool upsample, rten_resize_params* p) {
    memset(p, 0, sizeof(*p));
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

// MaxPool / AveragePool auto_pad (src/op_registry/onnx_registry.rs get_padding): NOTSET and VALID take the pads
// attribute, SAME_UPPER is `Padding::Same`; SAME_LOWER is refused as Conv refuses it
rten_status pool_auto_pad(rten_ctx* ctx, const onnx::Node& n, bool* same) {
    const onnx::Attribute* ap = n.attr("auto_pad");
    *same = ap && ap->s == "SAME_UPPER";
    if (ap && ap->s == "SAME_LOWER") return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "auto_pad SAME_LOWER is not supported");
    if (ap && !ap->s.empty() && ap->s != "NOTSET" && ap->s != "VALID" && ap->s != "SAME_UPPER")
        return mfail(ctx, RTEN_ERR_INVALID_VALUE, "auto_pad: unsupported value");
    return RTEN_OK;
}

// MaxPool / AveragePool attributes (kernel_shape, pads, strides, auto_pad, ceil_mode) for the NCHW input x, as pads under
// which the floor-rounded output size of the pooling entry points is the reference's (src/ops/pooling.rs
// output_size_and_padding_for_axis).  SAME_UPPER: the pads axis_out computes.  ceil_mode: the end pad that makes the
// floor formula give the ceil size, after the reference drops a last window that would start inside the end padding.
// Only the output size depends on the end pads: both pool kernels skip every tap outside the image, and divide by
// kh * kw under count_include_pad, as the reference's `average` does.
struct PoolAttrs {
    int32_t kernel[2], pads[4] = {0, 0, 0, 0}, strides[2] = {1, 1};
};
rten_status fill_pool_attrs(rten_ctx* ctx, const onnx::Node& n, const rten_tensor& x, PoolAttrs* a) {
    const std::vector<int64_t> k = n.attr_ints("kernel_shape"), pd = n.attr_ints("pads"), sd = n.attr_ints("strides");
    if (k.size() != 2) return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, n.op_type + ": only 2-D kernels are supported");
    if (x.ndim != 4) return mfail(ctx, RTEN_ERR_INVALID_VALUE, "input must have 4 dims (NCHW)");
    bool same = false;
    RTB_TRY(pool_auto_pad(ctx, n, &same));
    const bool ceil = n.attr_i("ceil_mode", 0) != 0;
    a->kernel[0] = (int32_t)k[0];
    a->kernel[1] = (int32_t)k[1];
    for (size_t i = 0; i < pd.size() && i < 4; i++) a->pads[i] = (int32_t)pd[i];
    for (size_t i = 0; i < sd.size() && i < 2; i++) a->strides[i] = (int32_t)sd[i];
    const int64_t in[2] = {x.shape[2], x.shape[3]};
    for (int i = 0; i < 2; i++) {
        int64_t out, ps, pe;
        RTB_TRY(api::axis_out(ctx, in[i], a->kernel[i], a->strides[i], same, a->pads[i], a->pads[2 + i], 1, &out, &ps, &pe));
        if (ceil && !same) {
            const int64_t s = a->strides[i], windows = in[i] + ps + pe - a->kernel[i];  // >= 0 past axis_out
            out = (windows + s - 1) / s + 1;
            if ((out - 1) * s >= in[i] + ps) out--;
            // floor((in + ps + pe' - k) / s) + 1 == out; 0 when the unpadded end already gives out windows
            pe = std::max<int64_t>(0, (out - 1) * s + a->kernel[i] - in[i] - ps);
        }
        a->pads[i] = (int32_t)ps;
        a->pads[2 + i] = (int32_t)pe;
    }
    return RTEN_OK;
}

// load checks of MaxPool / AveragePool: auto_pad, and MaxPool's Indices output, which the reference's MaxPool does not
// produce (max_outputs = 1)
template <bool max_pool>
rten_status check_pool(rten_model* m, onnx::Node& n) {
    bool same;
    RTB_TRY(pool_auto_pad(m->ctx, n, &same));
    if (max_pool && n.outputs.size() > 1 && !n.outputs[1].empty())
        return mfail(m->ctx, RTEN_ERR_UNSUPPORTED_VALUE, "MaxPool: the Indices output (1) is not supported");
    return RTEN_OK;
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

// ------------------------------------------------------------------------------------------
// run
// ------------------------------------------------------------------------------------------
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
    const rten_tensor* T(const OpNode& o, size_t i) { return (i < o.in.size() && o.in[i] >= 0) ? &V(o.in[i]).t : nullptr; }
    static bool wants(const OpNode& o, size_t k) { return k < o.out.size() && o.out[k] >= 0; }

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
        if (v.kind == V_INPUT) v.pending--;  // (only to know a writable input's last consumer)
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
    // output k of a node: the value's when the node names it, else the buffer goes back to the pool
    void set_output(const OpNode& o, size_t k, const rten_tensor& t) {
        if (wants(o, k)) set_owned(o.out[k], t);
        else pool_free(ctx, t.data);
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

    // output `id` as a run-time host value: `ints` in `shape` (no device memory, no launch)
    void set_host(int id, const std::vector<int64_t>& ints, int ndim, const int64_t* shape) {
        ValueSlot& v = V(id);
        v.has_host_ints = true;
        v.host_ints = ints;
        v.host_i32.assign(ints.size() ? ints.size() : 1, 0);
        for (size_t i = 0; i < ints.size(); i++) v.host_i32[i] = (int32_t)ints[i];
        rten_tensor t{};
        t.data = v.host_i32.data();
        t.dtype = RTEN_I32;
        t.ndim = ndim;
        for (int i = 0; i < ndim; i++) t.shape[i] = shape[i];
        set_contiguous(&t);
        t.device = RTEN_DEVICE_HOST;
        v.t = t;
        v.root = -1;
        v.live = true;
        v.owned = false;
    }

    // The attention cache input `slot` of node o extended in place (the reference's run_in_place, gqa_present_cache):
    // when it is a writable graph input whose grow axis is 2, this node is its last consumer, it is not a requested
    // output, the node wants present output `out_k` and the buffer holds grow more positions, `present` becomes the
    // past's buffer with the grown shape and true is returned.  Otherwise the node builds a new present cache.
    bool cache_in_place(const OpNode& o, size_t slot, size_t out_k, int64_t grow, rten_tensor* present) {
        if (slot >= o.in.size() || o.in[slot] < 0 || !wants(o, out_k)) return false;
        const ValueSlot& v = V(o.in[slot]);
        if (!v.writable || v.grow_axis != 2 || v.t.ndim != 4 || v.pending != 1 || keep.count(o.in[slot])) return false;
        if (v.t.shape[2] + grow > v.capacity) return false;
        *present = v.t;
        present->shape[2] += grow;
        return true;
    }
    // present output k of node o after the call: a view of the writable input it was written into, or a new buffer
    void set_present(const OpNode& o, size_t k, size_t slot, bool in_place, const rten_tensor& t) {
        if (!in_place) return set_output(o, k, t);
        set_view(o.out[k], t, o.in[slot]);
        V(o.out[k]).alias_of = V(o.in[slot]).input_index;
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
    rten_status resize_target(const OpNode& o, bool upsample, rten_resize_params* p) {
        RTB_TRY(fill_resize_params(ctx, o.n, upsample, p));
        const bool old = upsample || o.in.size() == 2;
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
        for (int i = 0; i < 4; i++) shape[i] = x.shape[i];
        return o.def->shape(*this, o, x, shape);
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

    // A view operator: its run function gives `y`, input 0 (made contiguous first for the ones that re-shape), its
    // shape and strides; no kernel runs
    rten_status run_view(OpNode& o) {
        rten_tensor y = V(o.in[0]).t;
        bool alloc = false;
        if (o.def->flags & RESHAPE) RTB_TRY(make_contiguous(V(o.in[0]).t, &y, &alloc));
        RTB_TRY(o.def->run(*this, o, &y));
        if (alloc) set_owned(o.out[0], y);
        else set_view(o.out[0], y, o.in[0]);
        // a view of a host-known value that keeps its element order stays host-known
        const ValueSlot& x = V(o.in[0]);
        if (x.has_host_ints && ((o.def->flags & RESHAPE) || std::string_view(o.def->name) == "Identity")) {
            ValueSlot& v = V(o.out[0]);
            v.has_host_ints = true;
            v.host_ints = x.host_ints;
        }
        return RTEN_OK;
    }

    // the contiguous `y` re-shaped to `shape`
    rten_status reshape(rten_tensor* y, const std::vector<int64_t>& shape) {
        int64_t prod = 1;
        for (int64_t d : shape) prod *= d;
        if (prod != numel(y)) return mfail(ctx, RTEN_ERR_INVALID_VALUE, "New shape must have same total elements as current shape");
        if ((int)shape.size() > RTEN_MAX_DIMS) return mfail(ctx, RTEN_ERR_INVALID_VALUE, "tensor rank out of range");
        y->ndim = (int)shape.size();
        for (int i = 0; i < y->ndim; i++) y->shape[i] = shape[(size_t)i];
        set_contiguous(y);
        return RTEN_OK;
    }

    // axes attribute (opset < 13) or second input
    rten_status axes_of(const OpNode& o, std::vector<int64_t>* axes) {
        *axes = o.n.attr_ints("axes");
        if (axes->empty() && o.in.size() > 1 && o.in[1] >= 0) RTB_TRY(ints_of(o.in[1], axes));
        return RTEN_OK;
    }

    rten_status run_node(OpNode& o) {
        const OpDef& d = *o.def;
        for (size_t i = 0; i < 32; i++)
            if ((d.required >> i & 1) && !T(o, i)) return mfail(ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
        if (d.flags & VIEW) return run_view(o);
        rten_tensor y;
        memset(&y, 0, sizeof(y));
        // in place when the executor holds the last reference to input 0 (src/graph.rs:973-1049)
        bool in_place = false;
        if (d.flags & IN_PLACE) {
            ValueSlot& x = V(o.in[0]);
            in_place = x.kind == V_TEMP && x.owned && x.root < 0 && x.pending == 1 && x.views == 0 && !keep.count(o.in[0]) && contiguous(x.t);
            if (in_place) y = x.t;
        }
        const bool into_concat = o.cat_node >= 0 && concat_slice(o, &y);
        RTB_TRY(d.run(*this, o, &y));
        if (in_place) {
            // the input's buffer now belongs to the output value
            ValueSlot& x = V(o.in[0]);
            x.owned = false;
            x.live = false;
        }
        if (into_concat)
            set_view(o.out[0], y, m->nodes[(size_t)o.cat_node].out[0]);
        else if (!wants(o, 0) || !V(o.out[0]).live)  // (a Cast that is a view, a Concat written in place: set already)
            set_output(o, 0, y);
        return RTEN_OK;
    }
};

// ---- the operators
rten_status prepack_conv(rten_ctx* ctx, OpNode& o, const rten_tensor& w) {
    return w.ndim == 4 ? rten_b200_prepack_conv_weight(ctx, &w, (int)o.n.attr_i("group", 1), &o.packed) : RTEN_OK;
}

rten_status prepack_matmul(rten_ctx* ctx, OpNode& o, const rten_tensor& w) {
    return w.ndim == 2 ? rten_b200_prepack_b(ctx, &w, &o.packed) : RTEN_OK;
}

// W [dirs, G * H, I] is the input projection's K-major B: prepack it as the [I, dirs * G * H] matrix
rten_status prepack_rnn(rten_ctx* ctx, OpNode& o, const rten_tensor& w0) {
    if (w0.dtype != RTEN_F32 || w0.ndim != 3) return RTEN_OK;
    rten_tensor w = w0;
    const int64_t rows = w.shape[0] * w.shape[1], I = w.shape[2];
    w.ndim = 2;
    w.shape[0] = I;
    w.shape[1] = rows;
    w.strides[0] = 1;
    w.strides[1] = I;
    return rten_b200_prepack_b(ctx, &w, &o.packed);
}

bool pool_shape(Runner& r, const OpNode& o, const rten_tensor& x, int64_t shape[4]) {
    PoolAttrs a;
    int64_t p0, p1;
    if (fill_pool_attrs(r.ctx, o.n, x, &a) != RTEN_OK) return false;
    for (int i = 0; i < 2; i++)
        if (api::axis_out(r.ctx, x.shape[2 + i], a.kernel[i], a.strides[i], false, a.pads[i], a.pads[2 + i], 1, &shape[2 + i], &p0, &p1) != RTEN_OK)
            return false;
    return true;
}

template <bool upsample>
rten_status run_resize(Runner& r, OpNode& o, rten_tensor* y) {
    rten_resize_params p;
    RTB_TRY(r.resize_target(o, upsample, &p));
    return rten_b200_resize(r.ctx, r.T(o, 0), &p, y);
}

template <bool upsample>
bool resize_shape(Runner& r, const OpNode& o, const rten_tensor& x, int64_t shape[4]) {
    rten_resize_params p;
    float inv[4];
    if (r.resize_target(o, upsample, &p) != RTEN_OK || api::resize_output_size(r.ctx, x, &p, shape, inv) != RTEN_OK) return false;
    return shape[0] == x.shape[0] && shape[1] == x.shape[1];
}

rten_status check_rms_norm(rten_model* m, onnx::Node& n) {  // onnx_registry.rs:1584-1590, 1905-1911
    if (n.attr_i("stash_type", 1) != 1) return mfail(m->ctx, RTEN_ERR_UNSUPPORTED_VALUE, n.op_type + ": stash_type must be 1");
    for (size_t i = 1; i < n.outputs.size(); i++)
        if (!n.outputs[i].empty())
            return mfail(m->ctx, RTEN_ERR_UNSUPPORTED_VALUE, n.op_type + ": only the normalized output (0) is supported");
    return RTEN_OK;
}

rten_status run_rms_norm(Runner& r, OpNode& o, rten_tensor* y) {
    return rten_b200_rms_norm(r.ctx, r.T(o, 0), r.T(o, 1), (int)o.n.attr_i("axis", -1), o.n.attr_f("epsilon", 1e-5f), y);
}

rten_status check_skip_norm(rten_model* m, onnx::Node& n) {  // onnx_registry.rs:1918-1932
    if (!n.attr("epsilon")) return mfail(m->ctx, RTEN_ERR_UNSUPPORTED_VALUE, n.op_type + ": missing attribute epsilon");
    // (the reference returns placeholder zeros for the training statistics, which no inference graph reads)
    for (size_t i = 1; i < 3 && i < n.outputs.size(); i++)
        if (!n.outputs[i].empty())
            return mfail(m->ctx, RTEN_ERR_UNSUPPORTED_VALUE, n.op_type + ": the mean and inv_std_var outputs (1, 2) are not supported");
    return RTEN_OK;
}

// inputs: x, skip, gamma, beta, bias (SkipLayerNormalization); x, skip, gamma, bias (the simplified one)
template <bool rms>
rten_status run_skip_norm(Runner& r, OpNode& o, rten_tensor* y) {
    rten_tensor s{};
    RTB_TRY(rten_b200_skip_layer_norm(r.ctx, r.T(o, 0), r.T(o, 1), r.T(o, 2), rms ? nullptr : r.T(o, 3), rms ? r.T(o, 3) : r.T(o, 4),
                                      o.n.attr_f("epsilon", 0.0f), rms ? 1 : 0, y, r.wants(o, 3) ? &s : nullptr));
    r.set_output(o, 3, s);
    return RTEN_OK;
}

// The shape a Reshape node with the constant target `target` gives `y`
rten_status reshape_target(Runner& r, int target, bool allowzero, const rten_tensor& y, std::vector<int64_t>* shape) {
    std::vector<int64_t> want;
    RTB_TRY(r.ints_of(target, &want));
    shape->clear();
    const int64_t total = numel(&y);
    int64_t known = 1;
    int infer = -1;
    for (size_t i = 0; i < want.size(); i++) {
        int64_t d = want[i];
        if (d == 0 && !allowzero) d = (int)i < y.ndim ? y.shape[i] : 0;
        if (d == -1) {
            if (infer >= 0) return mfail(r.ctx, RTEN_ERR_INVALID_VALUE, "Multiple dimensions in new shape set to -1");
            infer = (int)i;
            d = 1;
        }
        shape->push_back(d);
        known *= d;
    }
    if (infer >= 0) {
        if (known == 0 || total % known) return mfail(r.ctx, RTEN_ERR_INVALID_VALUE, "Input length must be a multiple of specified dimensions");
        (*shape)[(size_t)infer] = total / known;
    }
    return RTEN_OK;
}

// The GroupNorm chain the load fused (inputs x, inst_scale, inst_bias, gamma, beta, the two Reshape targets; the
// InstanceNormalization node's attributes).  The Reshapes' shapes are checked as they would resolve for this x, so an
// input the pattern does not fit fails with the message the node chain gives.
rten_status run_group_norm(Runner& r, OpNode& o, rten_tensor* y) {
    const rten_tensor* x = r.T(o, 0);
    const rten_tensor *gamma = r.T(o, 3), *beta = r.T(o, 4);
    const int64_t G = r.T(o, 1)->shape[0];
    std::vector<int64_t> s1, s2;
    rten_tensor v = *x;
    RTB_TRY(reshape_target(r, o.in[5], false, v, &s1));
    if ((int)s1.size() > RTEN_MAX_DIMS) return mfail(r.ctx, RTEN_ERR_INVALID_VALUE, "tensor rank out of range");
    v.ndim = (int)s1.size();
    for (int i = 0; i < v.ndim; i++) v.shape[i] = s1[(size_t)i];
    RTB_TRY(reshape_target(r, o.in[6], false, v, &s2));
    const bool grouped = x->ndim == 4 && s1.size() == 3 && s1[0] == x->shape[0] && s1[1] == G;
    if (!grouped || s2 != std::vector<int64_t>(x->shape, x->shape + 4))
        return mfail(r.ctx, RTEN_ERR_UNSUPPORTED_VALUE, "GroupNorm: the input does not fit the fused Reshape pattern");
    if (x->shape[1] != numel(gamma) || x->shape[1] != numel(beta))
        return mfail(r.ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "Cannot broadcast inputs");
    return rten_b200_group_norm(r.ctx, x, (int)G, r.T(o, 1), r.T(o, 2), gamma, beta, o.n.attr_f("epsilon", 1e-5f), &o.activation, y);
}

// ReduceSum (src/ops/reduce.rs:1116-1163) and ReduceMean (:543-580): axes from the attribute (opset < 13 / < 18) or
// input 1; none or empty reduces every axis, or, with noop_with_empty_axes, copies the input
template <bool MEAN>
rten_status run_reduce(Runner& r, OpNode& o, rten_tensor* y) {
    const rten_tensor* x = r.T(o, 0);
    std::vector<int64_t> axes;
    RTB_TRY(r.axes_of(o, &axes));
    if (axes.empty() && o.n.attr_i("noop_with_empty_axes", 0)) {
        rten_tensor c = *x;
        set_contiguous(&c);
        c.device = r.ctx->device;
        RTB_TRY(pool_alloc(r.ctx, (size_t)std::max<int64_t>(numel(&c), 1) * dtype_size(c.dtype), &c.data));
        const rten_status st = rten_b200_copy(r.ctx, x, &c);
        if (st != RTEN_OK) {
            pool_free(r.ctx, c.data);
            return st;
        }
        *y = c;
        return RTEN_OK;
    }
    std::vector<int32_t> a(axes.begin(), axes.end());
    return (MEAN ? rten_b200_reduce_mean : rten_b200_reduce_sum)(r.ctx, x, a.data(), (int)a.size(), (int)o.n.attr_i("keepdims", 1), y);
}

// TopK (src/ops/reduce.rs:1236-1306): K is input 1 (opset >= 10) or the `k` attribute (opset < 10).  A host-known K
// (a constant, or Shape -> Gather) costs nothing; a device-resident K is copied to the host and waited for, which
// keeps a step holding this node out of CUDA-graph capture.
rten_status run_topk(Runner& r, OpNode& o, rten_tensor* y) {
    int64_t k = 0;
    if (o.n.attr("k")) {
        k = o.n.attr_i("k", 0);
    } else {
        const rten_tensor* kt = r.T(o, 1);
        if (!kt) return mfail(r.ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
        if (numel(kt) != 1 || kt->dtype != RTEN_I32) return mfail(r.ctx, RTEN_ERR_INVALID_VALUE, "TopK: K must be one integer");
        const ValueSlot& kv = r.V(o.in[1]);
        if (kv.has_host_ints) {
            k = kv.host_ints[0];
        } else {
            int32_t hk = 0;
            RTB_CUDA(r.ctx, cudaMemcpyAsync(&hk, kt->data, 4, cudaMemcpyDeviceToHost, r.ctx->stream));
            RTB_CUDA(r.ctx, cudaStreamSynchronize(r.ctx->stream));
            k = hk;
        }
    }
    rten_tensor idx{};
    RTB_TRY(rten_b200_topk(r.ctx, r.T(o, 0), k, (int)o.n.attr_i("axis", -1), (int)o.n.attr_i("largest", 1),
                           (int)o.n.attr_i("sorted", 1), y, &idx));
    r.set_output(o, 1, idx);
    return RTEN_OK;
}

// ArgMax / ArgMin (src/op_registry/onnx_registry.rs get_common_arg_reduce_attrs): select_last_index must be 0
rten_status load_arg_reduce(rten_model* m, onnx::Node& n) {
    if (n.attr_i("select_last_index", 0) != 0)
        return mfail(m->ctx, RTEN_ERR_UNSUPPORTED_VALUE, n.op_type + ": select_last_index = 1 is not supported");
    return RTEN_OK;
}

// BatchNormalization (src/op_registry/onnx_registry.rs:830-842): inference mode only; momentum, a training attribute,
// is read and ignored as the reference does.  Outputs 1-4 are the training statistics (src/ops/norm.rs check_outputs).
rten_status check_batch_norm(rten_model* m, onnx::Node& n) {
    for (const char* a : {"training_mode", "spatial"})
        if (n.attr(a) && n.attr_i(a, 0) != (std::string_view(a) == "spatial" ? 1 : 0))
            return mfail(m->ctx, RTEN_ERR_UNSUPPORTED_VALUE, "BatchNormalization: error in attribute \"" + std::string(a) + "\": unsupported value");
    static const char* const stats[] = {"running_mean", "running_var", "saved_mean", "saved_var"};
    for (size_t i = 1; i < n.outputs.size() && i < 5; i++)
        if (!n.outputs[i].empty()) return mfail(m->ctx, RTEN_ERR_UNSUPPORTED_OUTPUT, std::string("unsupported output: ") + stats[i - 1]);
    return RTEN_OK;
}

rten_status run_batch_norm(Runner& r, OpNode& o, rten_tensor* y) {
    return rten_b200_batch_norm(r.ctx, r.T(o, 0), r.T(o, 1), r.T(o, 2), r.T(o, 3), r.T(o, 4), o.n.attr_f("epsilon", 1e-5f),
                                &o.activation, y);
}

// Shape (src/ops/layout.rs): the input's dims [start, end) -- negative from the end, clamped to [0, ndim], end at least
// start -- as a host value
rten_status run_shape(Runner& r, OpNode& o, rten_tensor*) {
    const rten_tensor* x = r.T(o, 0);
    const int64_t nd = x->ndim;
    auto bound = [&](const char* name, int64_t dflt) {
        if (!o.n.attr(name)) return dflt;
        const int64_t v = o.n.attr_i(name, 0);
        return std::min(nd, std::max<int64_t>(0, v < 0 ? v + nd : v));
    };
    const int64_t start = bound("start", 0), end = std::max(start, bound("end", nd));
    const std::vector<int64_t> dims(x->shape + start, x->shape + end);
    const int64_t n = (int64_t)dims.size();
    if (Runner::wants(o, 0)) r.set_host(o.out[0], dims, 1, &n);
    return RTEN_OK;
}

// Gather (src/ops/gather.rs gather) of a host-known vector on axis 0 with host-known indices (a scalar or a vector): a
// host value, negative indices from the end.  false: not such a Gather.
bool host_gather(Runner& r, OpNode& o, rten_status* st) {
    const ValueSlot& data = r.V(o.in[0]);
    const ValueSlot* idx = o.in.size() > 1 && o.in[1] >= 0 ? &r.V(o.in[1]) : nullptr;
    if (!data.has_host_ints || !idx || !idx->has_host_ints || data.t.ndim > 1 || idx->t.ndim > 1) return false;
    const int64_t axis = o.n.attr_i("axis", 0);
    if (data.t.ndim == 0 || (axis != 0 && axis != -1)) {
        *st = mfail(r.ctx, RTEN_ERR_INVALID_VALUE, "Axis is invalid");
        return true;
    }
    const int64_t len = data.t.shape[0];
    std::vector<int64_t> out;
    for (int64_t i : idx->host_ints) {
        const int64_t k = i < 0 ? i + len : i;
        if (k < 0 || k >= len) {
            *st = mfail(r.ctx, RTEN_ERR_INVALID_VALUE, "Entry in `indices` is out of range");
            return true;
        }
        out.push_back(data.host_ints[(size_t)k]);
    }
    if (Runner::wants(o, 0)) r.set_host(o.out[0], out, idx->t.ndim, idx->t.shape);
    *st = RTEN_OK;
    return true;
}

// ---- host values: shape arithmetic (the reference's i32 semantics)
// A host-known value's elements as the reference holds them: i32, an int64 constant saturated as the loader does
std::vector<int64_t> host_i32(const ValueSlot& v) {
    std::vector<int64_t> r(v.host_ints.size());
    for (size_t i = 0; i < r.size(); i++) r[i] = std::max<int64_t>(INT32_MIN, std::min<int64_t>(INT32_MAX, v.host_ints[i]));
    return r;
}

bool all_host(Runner& r, const OpNode& o, size_t n) {
    for (size_t i = 0; i < n; i++)
        if (i >= o.in.size() || o.in[i] < 0 || !r.V(o.in[i]).has_host_ints) return false;
    return true;
}

// The first n inputs of o, all host-known, broadcast together (numpy rules): `shape` and each input's elements at every
// output position
rten_status host_broadcast(Runner& r, const OpNode& o, size_t n, std::vector<int64_t>* shape, std::vector<std::vector<int64_t>>* vals) {
    int nd = 0;
    for (size_t i = 0; i < n; i++) nd = std::max(nd, r.V(o.in[i]).t.ndim);
    shape->assign((size_t)nd, 1);
    for (size_t i = 0; i < n; i++) {
        const rten_tensor& t = r.V(o.in[i]).t;
        for (int k = 0; k < t.ndim; k++) {
            int64_t& d = (*shape)[(size_t)(k + nd - t.ndim)];
            if (t.shape[k] != 1) {
                if (d != 1 && d != t.shape[k]) return mfail(r.ctx, RTEN_ERR_INCOMPATIBLE_SHAPES, "Cannot broadcast inputs");
                d = t.shape[k];
            }
        }
    }
    int64_t total = 1;
    for (int64_t d : *shape) total *= d;
    vals->assign(n, std::vector<int64_t>((size_t)total));
    for (size_t i = 0; i < n; i++) {
        const ValueSlot& v = r.V(o.in[i]);
        const std::vector<int64_t> src = host_i32(v);
        for (int64_t e = 0; e < total; e++) {
            int64_t rem = e, off = 0, st = 1;
            for (int k = nd - 1; k >= 0; k--) {
                const int64_t idx = rem % (*shape)[(size_t)k];
                rem /= (*shape)[(size_t)k];
                const int kk = k - (nd - v.t.ndim);
                if (kk >= 0) {
                    if (v.t.shape[kk] != 1) off += idx * st;
                    st *= v.t.shape[kk];
                }
            }
            (*vals)[i][(size_t)e] = src[(size_t)off];
        }
    }
    return RTEN_OK;
}

// f over the broadcast host inputs of o as its host output.  false: an input is not host-known (the node runs on the
// device).
template <size_t N, class F>
bool host_map(Runner& r, OpNode& o, rten_status* st, F f) {
    if (!all_host(r, o, N)) return false;
    std::vector<int64_t> shape;
    std::vector<std::vector<int64_t>> v;
    *st = host_broadcast(r, o, N, &shape, &v);
    if (*st != RTEN_OK) return true;
    std::vector<int64_t> out(v[0].size());
    for (size_t e = 0; e < out.size(); e++) {
        int64_t x[N];
        for (size_t i = 0; i < N; i++) x[i] = v[i][e];
        out[e] = f(x);
    }
    if (Runner::wants(o, 0)) r.set_host(o.out[0], out, (int)shape.size(), shape.data());
    *st = RTEN_OK;
    return true;
}

// Add / Sub / Mul wrap, Div truncates; a zero divisor (or INT_MIN / -1) fails as the device Div does
template <int OP>
bool host_arith(Runner& r, OpNode& o, rten_status* st) {
    // Div: every divisor is checked before the broadcast, as the reference's check_nonzero does; INT_MIN / -1 where the
    // two meet fails with the same message, as the device Div does
    if (OP == BIN_DIV && all_host(r, o, 2)) {
        bool bad = false;
        for (int64_t d : host_i32(r.V(o.in[1]))) bad = bad || d == 0;
        std::vector<int64_t> shape;
        std::vector<std::vector<int64_t>> v;
        if (!bad && host_broadcast(r, o, 2, &shape, &v) == RTEN_OK)
            for (size_t e = 0; e < v[0].size(); e++) bad = bad || (v[0][e] == INT32_MIN && v[1][e] == -1);
        if (bad) {
            *st = mfail(r.ctx, RTEN_ERR_INVALID_VALUE, "Divisor contains zero");
            return true;
        }
    }
    return host_map<2>(r, o, st, [](const int64_t* x) -> int64_t {
        const uint32_t a = (uint32_t)x[0], b = (uint32_t)x[1];
        if (OP == BIN_ADD) return (int32_t)(a + b);
        if (OP == BIN_SUB) return (int32_t)(a - b);
        if (OP == BIN_MUL) return (int32_t)(a * b);
        return (int32_t)(x[0] / x[1]);  // (no zero divisor, no INT_MIN / -1: refused above)
    });
}

template <int OP>
bool host_compare(Runner& r, OpNode& o, rten_status* st) {
    return host_map<2>(r, o, st, [](const int64_t* x) -> int64_t {
        switch (OP) {
            case CMP_EQ: return x[0] == x[1];
            case CMP_LT: return x[0] < x[1];
            case CMP_LE: return x[0] <= x[1];
            case CMP_GT: return x[0] > x[1];
            default: return x[0] >= x[1];
        }
    });
}

template <int OP>
rten_status run_compare(Runner& r, OpNode& o, rten_tensor* y) {
    rten_status st;
    if (host_compare<OP>(r, o, &st)) return st;
    auto fn = OP == CMP_EQ ? rten_b200_equal : OP == CMP_LT ? rten_b200_less : OP == CMP_LE ? rten_b200_less_or_equal
            : OP == CMP_GT ? rten_b200_greater : rten_b200_greater_or_equal;
    return fn(r.ctx, r.T(o, 0), r.T(o, 1), y);
}

// Concat on axis 0 of 1-D host values: a host value
bool host_concat(Runner& r, OpNode& o, rten_status* st) {
    if (o.in.empty() || !all_host(r, o, o.in.size())) return false;
    for (int i : o.in)
        if (r.V(i).t.ndim != 1) return false;
    if (o.n.attr_i("axis", 0) != 0 && o.n.attr_i("axis", 0) != -1) return false;
    std::vector<int64_t> out;
    for (int i : o.in) {
        const std::vector<int64_t> v = host_i32(r.V(i));
        out.insert(out.end(), v.begin(), v.end());
    }
    const int64_t n = (int64_t)out.size();
    if (Runner::wants(o, 0)) r.set_host(o.out[0], out, 1, &n);
    *st = RTEN_OK;
    return true;
}

// an i32 list input (host-known, saturated) or attribute `attr`; `present` false when neither is given
rten_status int_list(Runner& r, const OpNode& o, size_t slot, const char* attr, std::vector<int32_t>* v, bool* present) {
    v->clear();
    *present = false;
    if (slot < o.in.size() && o.in[slot] >= 0) {
        if (!r.V(o.in[slot]).has_host_ints)
            return mfail(r.ctx, RTEN_ERR_UNSUPPORTED_VALUE, o.n.op_type + ": input " + std::to_string(slot) + " must be known on the host");
        for (int64_t x : host_i32(r.V(o.in[slot]))) v->push_back((int32_t)x);
        *present = true;
    } else if (attr && o.n.attr(attr)) {
        for (int64_t x : o.n.attr_ints(attr)) v->push_back((int32_t)std::max<int64_t>(INT32_MIN, std::min<int64_t>(INT32_MAX, x)));
        *present = true;
    }
    return RTEN_OK;
}

// Slice (src/ops/slice.rs): a strided view of x (strides times the steps, an offset), no copy; of a 1-D host value, a
// host value.  Starts / ends / axes / steps are inputs (opset >= 10) or attributes (earlier), known on the host.
rten_status run_slice(Runner& r, OpNode& o, rten_tensor*) {
    const rten_tensor* x = r.T(o, 0);
    std::vector<int32_t> s, e, a, st;
    bool hs, he, ha, hst;
    RTB_TRY(int_list(r, o, 1, "starts", &s, &hs));
    RTB_TRY(int_list(r, o, 2, "ends", &e, &he));
    RTB_TRY(int_list(r, o, 3, "axes", &a, &ha));
    RTB_TRY(int_list(r, o, 4, nullptr, &st, &hst));
    if (!hs || !he) return mfail(r.ctx, RTEN_ERR_MISSING_INPUTS, "missing inputs");
    int64_t b[RTEN_MAX_DIMS], len[RTEN_MAX_DIMS], step[RTEN_MAX_DIMS];
    RTB_TRY(slice_ranges(r.ctx, x->ndim, x->shape, s.data(), (int)s.size(), e.data(), (int)e.size(), ha ? a.data() : nullptr, (int)a.size(),
                         hst ? st.data() : nullptr, (int)st.size(), b, len, step));
    if (!Runner::wants(o, 0)) return RTEN_OK;
    const ValueSlot& xv = r.V(o.in[0]);
    if (xv.has_host_ints && x->ndim == 1) {
        std::vector<int64_t> out;
        const std::vector<int64_t> src = host_i32(xv);
        for (int64_t i = 0; i < len[0]; i++) out.push_back(src[(size_t)(b[0] + i * step[0])]);
        r.set_host(o.out[0], out, 1, &len[0]);
        return RTEN_OK;
    }
    rten_tensor v = *x;
    for (int i = 0; i < x->ndim; i++) {
        if (len[i] > 0) v.data = (char*)v.data + b[i] * x->strides[i] * dtype_size(x->dtype);
        v.shape[i] = len[i];
        v.strides[i] = x->strides[i] * step[i];
    }
    r.set_view(o.out[0], v, o.in[0]);
    return RTEN_OK;
}

// Split (src/ops/split.rs): every output a view of its piece of x, no copy.  The sizes are input 1 (opset >= 13), the
// `split` attribute (earlier), else num_outputs (opset 18) or the node's output count pieces of ceil(n / k).
rten_status run_split(Runner& r, OpNode& o, rten_tensor*) {
    const rten_tensor* x = r.T(o, 0);
    const int64_t axis0 = o.n.attr_i("axis", 0), axis = axis0 < 0 ? axis0 + x->ndim : axis0;
    if (axis < 0 || axis >= x->ndim) return mfail(r.ctx, RTEN_ERR_INVALID_VALUE, "Axis is invalid");
    std::vector<int32_t> sizes;
    bool given;
    RTB_TRY(int_list(r, o, 1, "split", &sizes, &given));
    const int64_t k = o.n.attr("num_outputs") ? o.n.attr_i("num_outputs", 0) : (int64_t)o.out.size();
    std::vector<int64_t> pieces;
    RTB_TRY(split_pieces(r.ctx, x->shape[axis], given ? sizes.data() : nullptr, (int)sizes.size(), k, &pieces));
    // (an output without a piece would be read unset; a piece without an output would be dropped)
    if (pieces.size() / 2 != o.out.size())
        return mfail(r.ctx, RTEN_ERR_INVALID_VALUE, "Split: " + std::to_string(pieces.size() / 2) + " pieces for " +
                                                        std::to_string(o.out.size()) + " outputs");
    for (size_t i = 0; i < o.out.size(); i++) {
        if (!Runner::wants(o, i)) continue;
        rten_tensor v = *x;
        v.shape[axis] = pieces[2 * i + 1];
        if (v.shape[axis] > 0) v.data = (char*)v.data + pieces[2 * i] * x->strides[axis] * dtype_size(x->dtype);
        r.set_view(o.out[i], v, o.in[0]);
    }
    return RTEN_OK;
}

// one element of a Range input: host-known, else read back (a synchronisation)
rten_status range_scalar(Runner& r, int id, bool as_float, double* out) {
    const ValueSlot& v = r.V(id);
    if (numel(&v.t) != 1) return mfail(r.ctx, RTEN_ERR_INVALID_VALUE, "`start` must be a scalar");
    if (v.has_host_ints) *out = (double)host_i32(v)[0];
    else if (v.has_host_floats) *out = v.host_floats[0];
    else {
        uint32_t bits = 0;
        RTB_CUDA(r.ctx, cudaMemcpyAsync(&bits, v.t.data, 4, v.t.device < 0 ? cudaMemcpyHostToHost : cudaMemcpyDeviceToHost, r.ctx->stream));
        RTB_CUDA(r.ctx, cudaStreamSynchronize(r.ctx->stream));
        float f;
        int32_t i;
        memcpy(&f, &bits, 4);
        memcpy(&i, &bits, 4);
        *out = as_float ? (double)f : (double)i;
    }
    return RTEN_OK;
}

// Range (src/ops/generate.rs range): i32 gives a host value; f32 is computed on the host by the reference's serial
// `val = val + delta` in f32 and uploaded once
rten_status run_range(Runner& r, OpNode& o, rten_tensor* y) {
    const int dt = r.T(o, 0)->dtype;
    if (dt != RTEN_F32 && dt != RTEN_I32) return mfail(r.ctx, RTEN_ERR_UNSUPPORTED_TYPE, "unsupported type");
    double s, l, d;
    RTB_TRY(range_scalar(r, o.in[0], dt == RTEN_F32, &s));
    RTB_TRY(range_scalar(r, o.in[1], dt == RTEN_F32, &l));
    RTB_TRY(range_scalar(r, o.in[2], dt == RTEN_F32, &d));
    if (dt == RTEN_I32) {
        const int32_t limit = (int32_t)l, delta = (int32_t)d;
        if (delta == 0) return mfail(r.ctx, RTEN_ERR_INVALID_VALUE, "delta must be non-zero");
        std::vector<int64_t> out;
        for (int64_t v = (int32_t)s; (delta > 0 && v < limit) || (delta < 0 && v > limit); v += delta) out.push_back(v);
        const int64_t n = (int64_t)out.size();
        if (Runner::wants(o, 0)) r.set_host(o.out[0], out, 1, &n);
        return RTEN_OK;
    }
    const float limit = (float)l, delta = (float)d;
    if (delta == 0.0f) return mfail(r.ctx, RTEN_ERR_INVALID_VALUE, "delta must be non-zero");
    std::vector<float> out;
    for (float v = (float)s; (delta > 0.0f && v < limit) || (delta < 0.0f && v > limit); v = v + delta) out.push_back(v);
    rten_tensor t{};
    t.dtype = RTEN_F32;
    t.ndim = 1;
    t.shape[0] = (int64_t)out.size();
    set_contiguous(&t);
    t.device = r.ctx->device;
    RTB_TRY(pool_alloc(r.ctx, std::max<size_t>(out.size(), 1) * 4, &t.data));
    if (!out.empty()) {
        cudaError_t e = cudaMemcpyAsync(t.data, out.data(), out.size() * 4, cudaMemcpyHostToDevice, r.ctx->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(r.ctx->stream);  // (`out` goes away)
        if (e != cudaSuccess) {
            pool_free(r.ctx, t.data);
            return fail_cuda(r.ctx, e, "Range upload");
        }
    }
    *y = t;
    return RTEN_OK;
}

// ConstantOfShape (src/ops/generate.rs): the `value` attribute's one element (default f32 0) over the host-known shape;
// an integer fill is a host value, an f32 one a device fill
rten_status run_constant_of_shape(Runner& r, OpNode& o, rten_tensor* y) {
    std::vector<int32_t> dims;
    bool given;
    RTB_TRY(int_list(r, o, 0, nullptr, &dims, &given));
    std::vector<int64_t> shape;
    int64_t n = 1;
    for (int32_t d : dims) {
        if (d < 0) return mfail(r.ctx, RTEN_ERR_INVALID_VALUE, "Invalid shape");
        shape.push_back(d);
        n *= d;
    }
    if ((int)shape.size() > RTEN_MAX_DIMS) return mfail(r.ctx, RTEN_ERR_INVALID_VALUE, "tensor rank out of range");
    const onnx::Attribute* a = o.n.attr("value");
    int32_t type = onnx::DT_FLOAT;
    uint32_t bits = 0;
    if (a && a->has_t) {
        const onnx::Tensor& t = a->t;
        if (t.numel() != 1) return mfail(r.ctx, RTEN_ERR_INVALID_VALUE, "ConstantOfShape: value must have one element");
        type = t.data_type;
        if (type == onnx::DT_INT64) {
            int64_t v;
            memcpy(&v, t.data.data(), 8);
            bits = (uint32_t)(int32_t)std::max<int64_t>(INT32_MIN, std::min<int64_t>(INT32_MAX, v));
        } else if (type == onnx::DT_INT32 || type == onnx::DT_FLOAT) {
            memcpy(&bits, t.data.data(), 4);
        } else if (type == onnx::DT_BOOL) {
            bits = t.data[0] ? 1 : 0;
        } else {
            return mfail(r.ctx, RTEN_ERR_UNSUPPORTED_TYPE, "ConstantOfShape: unsupported value type");
        }
    }
    if (type != onnx::DT_FLOAT) {
        if (Runner::wants(o, 0)) r.set_host(o.out[0], std::vector<int64_t>((size_t)n, (int64_t)(int32_t)bits), (int)shape.size(), shape.data());
        return RTEN_OK;
    }
    rten_tensor t{};
    t.dtype = RTEN_F32;
    t.ndim = (int)shape.size();
    for (int i = 0; i < t.ndim; i++) t.shape[i] = shape[(size_t)i];
    set_contiguous(&t);
    t.device = r.ctx->device;
    RTB_TRY(pool_alloc(r.ctx, (size_t)std::max<int64_t>(n, 1) * 4, &t.data));
    const rten_status st = launch_fill(r.ctx, t.data, bits, n);
    if (st != RTEN_OK) {
        pool_free(r.ctx, t.data);
        return st;
    }
    *y = t;
    return RTEN_OK;
}

// Where: of host-known inputs a host value, else on the device
rten_status run_where(Runner& r, OpNode& o, rten_tensor* y) {
    rten_status st;
    if (host_map<3>(r, o, &st, [](const int64_t* x) { return x[0] != 0 ? x[1] : x[2]; })) return st;
    return rten_b200_where(r.ctx, r.T(o, 0), r.T(o, 1), r.T(o, 2), y);
}

rten_status run_expand(Runner& r, OpNode& o, rten_tensor* y) {
    std::vector<int32_t> dims;
    bool given;
    RTB_TRY(int_list(r, o, 1, nullptr, &dims, &given));
    const std::vector<int64_t> shape(dims.begin(), dims.end());
    return rten_b200_expand(r.ctx, r.T(o, 0), shape.data(), (int)shape.size(), y);
}

rten_status run_trilu(Runner& r, OpNode& o, rten_tensor* y) {
    std::vector<int32_t> k;
    bool given;
    RTB_TRY(int_list(r, o, 1, nullptr, &k, &given));
    if (given && k.size() != 1) return mfail(r.ctx, RTEN_ERR_INVALID_VALUE, "k must be a scalar");
    return rten_b200_trilu(r.ctx, r.T(o, 0), given ? k[0] : 0, (int)o.n.attr_i("upper", 1), y);
}

constexpr OpDef OPS[] = {
    {"Conv", ONNX, 0, 0b1, [](Runner& r, OpNode& o, rten_tensor* y) {
         rten_conv_params p;
         RTB_TRY(fill_conv_params(r.ctx, o.n, &p));
         return rten_b200_conv2d_act(r.ctx, r.T(o, 0), r.T(o, 1), o.packed, r.T(o, 2), &p, nullptr, &o.activation, y);
     }, nullptr, prepack_conv, [](Runner& r, const OpNode& o, const rten_tensor& x, int64_t shape[4]) {
         const rten_tensor* w = r.T(o, 1);
         rten_conv_params p;
         int64_t p0, p1;
         if (!w || w->ndim != 4 || fill_conv_params(r.ctx, o.n, &p) != RTEN_OK) return false;
         shape[1] = w->shape[0];
         for (int a = 0; a < 2; a++)
             if (api::axis_out(r.ctx, x.shape[2 + a], w->shape[2 + a], p.strides[a], p.auto_pad_same != 0, p.pads[a], p.pads[2 + a],
                               p.dilations[a], &shape[2 + a], &p0, &p1) != RTEN_OK)
                 return false;
         return true;
     }},
    {"ConvInteger", ONNX, 0, 0b1, [](Runner& r, OpNode& o, rten_tensor* y) {
         rten_conv_params p;
         RTB_TRY(fill_conv_params(r.ctx, o.n, &p));
         return rten_b200_conv_integer(r.ctx, r.T(o, 0), r.T(o, 1), o.packed, r.T(o, 2), r.T(o, 3), nullptr, &p, y);
     }, nullptr, prepack_conv},
    {"ConvTranspose", ONNX, 0, 0b1, [](Runner& r, OpNode& o, rten_tensor* y) {
         rten_conv_transpose_params p;
         RTB_TRY(fill_conv_transpose_params(r.ctx, o.n, &p));
         return rten_b200_conv_transpose(r.ctx, r.T(o, 0), r.T(o, 1), o.packed, r.T(o, 2), &p, y);
     }, [](rten_model* m, onnx::Node& n) {  // (the reference does not read output_shape)
         return !n.attr("output_shape") ? RTEN_OK : mfail(m->ctx, RTEN_ERR_UNSUPPORTED_VALUE, "ConvTranspose: the output_shape attribute is not supported");
     }, [](rten_ctx* ctx, OpNode& o, const rten_tensor& w) {
         if (w.dtype != RTEN_F32) return RTEN_OK;
         // (a weight whose attributes the operator would refuse is not prepacked: the run reports the error)
         rten_conv_transpose_params p;
         RTB_TRY(fill_conv_transpose_params(ctx, o.n, &p));
         if (rten_b200_prepack_conv_transpose_weight(ctx, &w, &p, &o.packed) != RTEN_OK) o.packed = nullptr;
         return RTEN_OK;
     }, [](Runner& r, const OpNode& o, const rten_tensor& x, int64_t shape[4]) {
         const rten_tensor* w = r.T(o, 1);
         rten_conv_transpose_params p;
         api::ConvTShape S;
         if (!w || fill_conv_transpose_params(r.ctx, o.n, &p) != RTEN_OK || api::conv_transpose_shape(r.ctx, &x, *w, nullptr, &p, S) != RTEN_OK)
             return false;
         shape[1] = S.O, shape[2] = S.OH, shape[3] = S.OW;
         return true;
     }},
    {"Relu", ONNX, IN_PLACE, 0b1, [](Runner& r, OpNode& o, rten_tensor* y) { return rten_b200_relu(r.ctx, r.T(o, 0), y); }, nullptr, nullptr, nullptr, RTEN_ACT_RELU},
    {"Clip", ONNX, IN_PLACE, 0b1, [](Runner& r, OpNode& o, rten_tensor* y) { return rten_b200_clip(r.ctx, r.T(o, 0), r.T(o, 1), r.T(o, 2), y); },
     [](rten_model* m, onnx::Node& n) {
         RTB_TRY(attr_to_input(m, n, "min", 1, "clip_min", true));
         return attr_to_input(m, n, "max", 2, "clip_max", true);
     }},
    {"Sigmoid", ONNX, IN_PLACE, 0b1, [](Runner& r, OpNode& o, rten_tensor* y) { return rten_b200_sigmoid(r.ctx, r.T(o, 0), y); }, nullptr, nullptr, nullptr, RTEN_ACT_SIGMOID},
    {"Silu", 0, IN_PLACE, 0b1, [](Runner& r, OpNode& o, rten_tensor* y) { return rten_b200_silu(r.ctx, r.T(o, 0), y); }, nullptr, nullptr, nullptr, RTEN_ACT_SILU},  // (SiluFusion)
    {"HardSigmoid", ONNX, IN_PLACE, 0b1, [](Runner& r, OpNode& o, rten_tensor* y) {
         return rten_b200_hard_sigmoid(r.ctx, r.T(o, 0), hard_sigmoid_alpha(o.n), hard_sigmoid_beta(o.n), y); }, nullptr, nullptr, nullptr, RTEN_ACT_HARD_SIGMOID},
    {"HardSwish", ONNX, IN_PLACE, 0b1, [](Runner& r, OpNode& o, rten_tensor* y) { return rten_b200_hard_swish(r.ctx, r.T(o, 0), y); }, nullptr, nullptr, nullptr, RTEN_ACT_HARD_SWISH},
    {"Gelu", ONNX | MS, IN_PLACE, 0b1, [](Runner& r, OpNode& o, rten_tensor* y) {
         const onnx::Attribute* a = o.n.attr("approximate");
         return rten_b200_gelu(r.ctx, r.T(o, 0), (a && a->s == "tanh") ? 1 : 0, y);
     }},
    {"Erf", ONNX, IN_PLACE, 0b1, [](Runner& r, OpNode& o, rten_tensor* y) { return rten_b200_erf(r.ctx, r.T(o, 0), y); }},
    {"Sqrt", ONNX, IN_PLACE, 0b1, [](Runner& r, OpNode& o, rten_tensor* y) { return rten_b200_sqrt(r.ctx, r.T(o, 0), y); }},
    {"Reciprocal", ONNX, IN_PLACE, 0b1, [](Runner& r, OpNode& o, rten_tensor* y) { return rten_b200_reciprocal(r.ctx, r.T(o, 0), y); }},
    {"Exp", ONNX, IN_PLACE, 0b1, [](Runner& r, OpNode& o, rten_tensor* y) { return rten_b200_exp(r.ctx, r.T(o, 0), y); }},
    {"Tanh", ONNX, IN_PLACE, 0b1, [](Runner& r, OpNode& o, rten_tensor* y) { return rten_b200_tanh(r.ctx, r.T(o, 0), y); }},
    {"Neg", ONNX, IN_PLACE, 0b1, [](Runner& r, OpNode& o, rten_tensor* y) { return rten_b200_neg(r.ctx, r.T(o, 0), y); }},
    {"Abs", ONNX, IN_PLACE, 0b1, [](Runner& r, OpNode& o, rten_tensor* y) { return rten_b200_abs(r.ctx, r.T(o, 0), y); }},
    {"Softmax", ONNX, IN_PLACE, 0b1, [](Runner& r, OpNode& o, rten_tensor* y) { return rten_b200_softmax(r.ctx, r.T(o, 0), nullptr, (int)o.n.attr_i("axis", -1), 0, y); }},
    {"MaxPool", ONNX, 0, 0b1, [](Runner& r, OpNode& o, rten_tensor* y) {
         PoolAttrs a;
         RTB_TRY(fill_pool_attrs(r.ctx, o.n, *r.T(o, 0), &a));
         return rten_b200_max_pool(r.ctx, r.T(o, 0), a.kernel, a.pads, a.strides, y);
     }, check_pool<true>, nullptr, pool_shape},
    {"AveragePool", ONNX, 0, 0b1, [](Runner& r, OpNode& o, rten_tensor* y) {
         PoolAttrs a;
         RTB_TRY(fill_pool_attrs(r.ctx, o.n, *r.T(o, 0), &a));
         return rten_b200_average_pool(r.ctx, r.T(o, 0), a.kernel, a.pads, a.strides, (int)o.n.attr_i("count_include_pad", 0), y);
     }, check_pool<false>, nullptr, pool_shape},
    {"Resize", ONNX, 0, 0b1, run_resize<false>, [](rten_model* m, onnx::Node& n) { rten_resize_params p; return fill_resize_params(m->ctx, n, false, &p); },
     nullptr, resize_shape<false>},
    {"Upsample", ONNX, 0, 0b1, run_resize<true>, [](rten_model* m, onnx::Node& n) {
         rten_resize_params p;
         RTB_TRY(fill_resize_params(m->ctx, n, true, &p));
         return attr_to_input(m, n, "scales", 1, "upsample_scales", false);
     }, nullptr, resize_shape<true>},
    {"Concat", ONNX, 0, 0b1, [](Runner& r, OpNode& o, rten_tensor* y) {
         rten_status st;
         if (host_concat(r, o, &st)) return st;
         std::vector<const rten_tensor*> ins;
         for (size_t i = 0; i < o.in.size(); i++)
             if (r.T(o, i)) ins.push_back(r.T(o, i));
         auto cs = r.cats.find((int)(&o - r.m->nodes.data()));
         // written in place: the buffer is the output value already; inputs that are their slice of it are skipped
         rten_tensor* out = cs != r.cats.end() && cs->second.active ? &cs->second.buf : y;
         return rten_b200_concat(r.ctx, ins.data(), (int)ins.size(), (int)o.n.attr_i("axis", 0), out);
     }, [](rten_model* m, onnx::Node& n) {
         return n.attr("axis") ? RTEN_OK : mfail(m->ctx, RTEN_ERR_UNSUPPORTED_VALUE, "Concat: missing attribute axis");
     }},
    {"GlobalAveragePool", ONNX, 0, 0b1, [](Runner& r, OpNode& o, rten_tensor* y) { return rten_b200_global_average_pool(r.ctx, r.T(o, 0), y); }},
    {"ReduceSum", ONNX, 0, 0b1, run_reduce<false>},
    {"TopK", ONNX, 0, 0b1, run_topk},
    {"ArgMax", ONNX, 0, 0b1, [](Runner& r, OpNode& o, rten_tensor* y) {
         return rten_b200_arg_max(r.ctx, r.T(o, 0), (int)o.n.attr_i("axis", 0), (int)o.n.attr_i("keepdims", 1), y); },
     load_arg_reduce},
    {"ArgMin", ONNX, 0, 0b1, [](Runner& r, OpNode& o, rten_tensor* y) {
         return rten_b200_arg_min(r.ctx, r.T(o, 0), (int)o.n.attr_i("axis", 0), (int)o.n.attr_i("keepdims", 1), y); },
     load_arg_reduce},
    {"Shape", ONNX, 0, 0b1, run_shape},
    {"ReduceMean", ONNX, 0, 0b1, [](Runner& r, OpNode& o, rten_tensor* y) {
         const rten_tensor* x = r.T(o, 0);
         std::vector<int64_t> axes;
         RTB_TRY(r.axes_of(o, &axes));
         bool spatial = x->ndim == 4 && axes.size() == 2;
         for (int64_t a : axes) {
             const int64_t p = a < 0 ? a + x->ndim : a;
             if (p != 2 && p != 3) spatial = false;
         }
         if (!spatial) return run_reduce<true>(r, o, y);
         RTB_TRY(rten_b200_global_average_pool(r.ctx, x, y));
         if (o.n.attr_i("keepdims", 1) == 0) {
             y->ndim = 2;
             set_contiguous(y);
         }
         return RTEN_OK;
     }},
    {"Reshape", ONNX, VIEW | RESHAPE, 0b1, [](Runner& r, OpNode& o, rten_tensor* y) {
         std::vector<int64_t> shape;
         RTB_TRY(reshape_target(r, o.in.size() > 1 ? o.in[1] : -1, o.n.attr_i("allowzero", 0) != 0, *y, &shape));
         return r.reshape(y, shape);
     }},
    {"Flatten", ONNX, VIEW | RESHAPE, 0b1, [](Runner& r, OpNode& o, rten_tensor* y) {
         int64_t axis = o.n.attr_i("axis", 1), a = 1, b = 1;
         if (axis < 0) axis += y->ndim;
         for (int i = 0; i < y->ndim; i++) (i < axis ? a : b) *= y->shape[i];
         return r.reshape(y, {a, b});
     }},
    {"Squeeze", ONNX, VIEW | RESHAPE, 0b1, [](Runner& r, OpNode& o, rten_tensor* y) {
         std::vector<int64_t> axes, shape;
         RTB_TRY(r.axes_of(o, &axes));
         for (int i = 0; i < y->ndim; i++) {
             bool drop = axes.empty() ? y->shape[i] == 1 : false;
             for (int64_t a : axes)
                 if ((a < 0 ? a + y->ndim : a) == i) drop = true;
             if (!drop) shape.push_back(y->shape[i]);
         }
         return r.reshape(y, shape);
     }},
    {"Unsqueeze", ONNX, VIEW | RESHAPE, 0b1, [](Runner& r, OpNode& o, rten_tensor* y) {
         std::vector<int64_t> axes, shape;
         RTB_TRY(r.axes_of(o, &axes));
         const int nd = y->ndim + (int)axes.size();
         std::vector<bool> ins((size_t)nd, false);
         for (int64_t a : axes) {
             const int64_t p = a < 0 ? a + nd : a;
             if (p < 0 || p >= nd) return mfail(r.ctx, RTEN_ERR_INVALID_VALUE, "Axes must be in range [-r, r-1]");
             ins[(size_t)p] = true;
         }
         int k = 0;
         for (int i = 0; i < nd; i++) shape.push_back(ins[(size_t)i] ? 1 : y->shape[k++]);
         return r.reshape(y, shape);
     }},
    {"Transpose", ONNX, VIEW, 0b1, [](Runner& r, OpNode& o, rten_tensor* y) {
         const rten_tensor x = *y;
         std::vector<int64_t> perm = o.n.attr_ints("perm");
         if (perm.empty())
             for (int i = x.ndim - 1; i >= 0; i--) perm.push_back(i);
         if ((int)perm.size() != x.ndim) return mfail(r.ctx, RTEN_ERR_INVALID_VALUE, "Transpose: perm has the wrong length");
         for (int i = 0; i < x.ndim; i++) {
             const int64_t a = perm[(size_t)i];
             if (a < 0 || a >= x.ndim) return mfail(r.ctx, RTEN_ERR_INVALID_VALUE, "Transpose: perm entry out of range");
             y->shape[i] = x.shape[a];
             y->strides[i] = x.strides[a];
         }
         return RTEN_OK;
     }},
    {"Identity", ONNX, VIEW, 0b1, [](Runner&, OpNode&, rten_tensor*) { return RTEN_OK; }},
    {"Gemm", ONNX, 0, 0b1, [](Runner& r, OpNode& o, rten_tensor* y) {
         return rten_b200_gemm(r.ctx, r.T(o, 0), r.T(o, 1), r.T(o, 2), o.n.attr_f("alpha", 1.0f), o.n.attr_f("beta", 1.0f),
                               (int)o.n.attr_i("transA", 0), (int)o.n.attr_i("transB", 0), y);
     }},
    {"MatMul", ONNX, 0, 0b1, [](Runner& r, OpNode& o, rten_tensor* y) {
         const rten_tensor* bias = o.bias_value >= 0 ? &r.V(o.bias_value).t : nullptr;
         return rten_b200_matmul(r.ctx, r.T(o, 0), r.T(o, 1), o.packed, bias, 1.0f, y);
     }, nullptr, prepack_matmul},
    {"MatMulInteger", ONNX, 0, 0b1, [](Runner& r, OpNode& o, rten_tensor* y) {
         return rten_b200_matmul_integer(r.ctx, r.T(o, 0), r.T(o, 1), o.packed, r.T(o, 2), r.T(o, 3), nullptr, y); }, nullptr, prepack_matmul},
    {"MatMulNBits", MS, 0, 0b111, [](Runner& r, OpNode& o, rten_tensor* y) {
         // accuracy_level only sets a minimum: every level computes in f32 (src/ops/matmul/contrib.rs:104-109)
         if (o.in.size() > 3) return mfail(r.ctx, RTEN_ERR_UNSUPPORTED_VALUE, "zero_points, g_idx and bias inputs are unsupported");
         return rten_b200_matmul_nbits(r.ctx, r.T(o, 0), r.T(o, 1), r.T(o, 2), 4, (int)o.n.attr_i("block_size", 0), y);
     }, [](rten_model* m, onnx::Node& n) {  // src/op_registry/onnx_registry.rs:1376-1402
         if (n.attr_i("bits", 4) != 4) return mfail(m->ctx, RTEN_ERR_UNSUPPORTED_VALUE, "MatMulNBits: only bits = 4 is supported");
         if (!n.attr("block_size")) return mfail(m->ctx, RTEN_ERR_UNSUPPORTED_VALUE, "MatMulNBits: missing attribute block_size");
         return RTEN_OK;
     }},
    {"Add", ONNX, 0, 0b11, [](Runner& r, OpNode& o, rten_tensor* y) {
         rten_status st;
         if (host_arith<BIN_ADD>(r, o, &st)) return st;
         return rten_b200_add(r.ctx, r.T(o, 0), r.T(o, 1), y);
     }},
    {"Sub", ONNX, 0, 0b11, [](Runner& r, OpNode& o, rten_tensor* y) {
         rten_status st;
         if (host_arith<BIN_SUB>(r, o, &st)) return st;
         return rten_b200_sub(r.ctx, r.T(o, 0), r.T(o, 1), y);
     }},
    {"Mul", ONNX, 0, 0b11, [](Runner& r, OpNode& o, rten_tensor* y) {
         rten_status st;
         if (host_arith<BIN_MUL>(r, o, &st)) return st;
         return rten_b200_mul(r.ctx, r.T(o, 0), r.T(o, 1), y);
     }},
    {"Div", ONNX, 0, 0b11, [](Runner& r, OpNode& o, rten_tensor* y) {
         rten_status st;
         if (host_arith<BIN_DIV>(r, o, &st)) return st;
         return rten_b200_div(r.ctx, r.T(o, 0), r.T(o, 1), y);
     }},
    {"Pow", ONNX, 0, 0b11, [](Runner& r, OpNode& o, rten_tensor* y) { return rten_b200_pow(r.ctx, r.T(o, 0), r.T(o, 1), y); }},
    {"LayerNormalization", ONNX, 0, 0b1, [](Runner& r, OpNode& o, rten_tensor* y) {
         return rten_b200_layer_norm(r.ctx, r.T(o, 0), r.T(o, 1), r.T(o, 2), (int)o.n.attr_i("axis", -1), o.n.attr_f("epsilon", 1e-5f), y); }},
    {"RMSNormalization", ONNX, 0, 0b11, run_rms_norm, check_rms_norm},
    {"SimplifiedLayerNormalization", ONNX, 0, 0b11, run_rms_norm, check_rms_norm},
    {"InstanceNormalization", ONNX, IN_PLACE, 0b111, [](Runner& r, OpNode& o, rten_tensor* y) {
         return rten_b200_instance_norm(r.ctx, r.T(o, 0), r.T(o, 1), r.T(o, 2), o.n.attr_f("epsilon", 1e-5f), y); }},
    {"GroupNorm", 0, IN_PLACE, 0b1111111, run_group_norm},  // (GroupNormFusion)
    {"BatchNormalization", ONNX, IN_PLACE, 0b11111, run_batch_norm, check_batch_norm},
    {"SkipLayerNormalization", MS, 0, 0b1, run_skip_norm<false>, check_skip_norm},
    {"SkipSimplifiedLayerNormalization", MS, 0, 0b1, run_skip_norm<true>, check_skip_norm},
    {"Gather", ONNX, 0, 0b1, [](Runner& r, OpNode& o, rten_tensor* y) {
         rten_status st;
         if (host_gather(r, o, &st)) return st;
         if (o.n.attr_i("axis", 0) != 0 || r.T(o, 0)->ndim != 2)
             return mfail(r.ctx, RTEN_ERR_UNSUPPORTED_VALUE, "Gather: only axis 0 of a 2-D table is supported");
         return rten_b200_gather_rows(r.ctx, r.T(o, 0), r.T(o, 1), y);
     }},
    {"Cast", ONNX, 0, 0b1, [](Runner& r, OpNode& o, rten_tensor* y) {
         const int64_t to = o.n.attr_i("to", 0);
         const rten_tensor* x = r.T(o, 0);
         const bool to_int = to == onnx::DT_INT32 || to == onnx::DT_INT64 || to == onnx::DT_BOOL;  // (bool is i32)
         if ((to == onnx::DT_FLOAT && x->dtype == RTEN_F32) || (to_int && x->dtype == RTEN_I32)) {
             r.set_view(o.out[0], *x, o.in[0]);
             if (to_int && r.V(o.in[0]).has_host_ints) {  // (stays host-known)
                 ValueSlot& v = r.V(o.out[0]);
                 v.has_host_ints = true;
                 v.host_ints = r.V(o.in[0]).host_ints;
                 if (to == onnx::DT_INT32)
                     for (int64_t& i : v.host_ints) i = (int32_t)i;
             }
             return RTEN_OK;
         }
         if (to != onnx::DT_FLOAT || x->dtype != RTEN_I32) return mfail(r.ctx, RTEN_ERR_UNSUPPORTED_VALUE, "Cast: only int32 -> float is supported");
         rten_tensor c;
         bool alloc = false;
         if (x->device < 0) {  // a host value: uploaded first
             c = *x;
             set_contiguous(&c);
             c.device = r.ctx->device;
             RTB_TRY(pool_alloc(r.ctx, (size_t)std::max<int64_t>(numel(x), 1) * 4, &c.data));
             alloc = true;
             const rten_status st = rten_b200_copy(r.ctx, x, &c);
             if (st != RTEN_OK) {
                 pool_free(r.ctx, c.data);
                 return st;
             }
         } else {
             RTB_TRY(r.make_contiguous(*x, &c, &alloc));
         }
         *y = c;
         y->dtype = RTEN_F32;
         void* d = nullptr;
         rten_status st = pool_alloc(r.ctx, (size_t)std::max<int64_t>(numel(&c), 1) * 4, &d);
         if (st == RTEN_OK) {
             y->data = d;
             st = launch_cast_scale(r.ctx, (const int*)c.data, (float*)d, numel(&c), 1, r.m->one, 1);  // f32(x) * 1.0f: exact
         }
         if (alloc) pool_free(r.ctx, c.data);
         return st;
     }},
    {"DynamicQuantizeLinear", ONNX, 0, 0b1, [](Runner& r, OpNode& o, rten_tensor* y) {
         rten_tensor s{}, z{};
         RTB_TRY(rten_b200_dynamic_quantize_linear(r.ctx, r.T(o, 0), y, &s, &z, nullptr));
         r.set_output(o, 1, s);
         r.set_output(o, 2, z);
         return RTEN_OK;
     }},
    {"Attention", ONNX, 0, 0b1, [](Runner& r, OpNode& o, rten_tensor* y) {
         rten_attention_params p;
         memset(&p, 0, sizeof(p));
         p.is_causal = (int32_t)o.n.attr_i("is_causal", 0);
         p.q_num_heads = (int32_t)o.n.attr_i("q_num_heads", 0);
         p.kv_num_heads = (int32_t)o.n.attr_i("kv_num_heads", 0);
         p.scale = o.n.attr_f("scale", 0.0f);
         p.softcap = o.n.attr_f("softcap", 0.0f);
         if (r.T(o, 4) || r.T(o, 5))
             return mfail(r.ctx, RTEN_ERR_UNSUPPORTED_VALUE, "Attention: past_key / past_value inputs are not supported by the executor");
         return rten_b200_attention(r.ctx, r.T(o, 0), r.T(o, 1), r.T(o, 2), r.T(o, 3), r.T(o, 6), &p, nullptr, nullptr, y);
     }},
    {"RotaryEmbedding", ONNX, 0, 0b111, [](Runner& r, OpNode& o, rten_tensor* y) {
         return rten_b200_rotary_embedding(r.ctx, r.T(o, 0), r.T(o, 1), r.T(o, 2), r.T(o, 3), (int)o.n.attr_i("interleaved", 0),
                                           (int)o.n.attr_i("num_heads", 0), (int)o.n.attr_i("rotary_embedding_dim", 0), y);
     }},
    {"GroupQueryAttention", MS, 0, 0b1100001, [](Runner& r, OpNode& o, rten_tensor* y) {
         if (r.T(o, 11)) return mfail(r.ctx, RTEN_ERR_UNSUPPORTED_VALUE, "head_sink is not supported");
         if (o.n.attr_i("smooth_softmax", 0)) return mfail(r.ctx, RTEN_ERR_UNSUPPORTED_VALUE, "smooth_softmax is not supported");
         rten_gqa_params p;
         memset(&p, 0, sizeof(p));
         p.num_heads = (int32_t)o.n.attr_i("num_heads", 0);
         p.kv_num_heads = (int32_t)o.n.attr_i("kv_num_heads", 0);
         p.scale = o.n.attr_f("scale", 0.0f);
         p.do_rotary = (int32_t)o.n.attr_i("do_rotary", 0);
         p.rotary_interleaved = (int32_t)o.n.attr_i("rotary_interleaved", 0);
         p.local_window_size = (int32_t)o.n.attr_i("local_window_size", -1);
         p.softcap = o.n.attr_f("softcap", 0.0f);
         rten_tensor pk{}, pv{};
         const int64_t S = r.T(o, 0)->ndim >= 2 ? r.T(o, 0)->shape[1] : 0;
         const bool ik = r.cache_in_place(o, 3, 1, S, &pk), iv = r.cache_in_place(o, 4, 2, S, &pv);
         RTB_TRY(rten_b200_group_query_attention(r.ctx, r.T(o, 0), r.T(o, 1), r.T(o, 2), r.T(o, 3), r.T(o, 4), r.T(o, 5), r.T(o, 6),
                                                 r.T(o, 7), r.T(o, 8), r.T(o, 9), r.T(o, 10), &p, y, &pk, &pv));
         r.set_present(o, 1, 3, ik, pk);
         r.set_present(o, 2, 4, iv, pv);
         return RTEN_OK;
     }, [](rten_model* m, onnx::Node& n) {  // src/op_registry/onnx_registry.rs:1467-1492, contrib.rs:817-821
         if (!n.attr("num_heads") || !n.attr("kv_num_heads"))
             return mfail(m->ctx, RTEN_ERR_UNSUPPORTED_VALUE, "GroupQueryAttention: missing attribute num_heads or kv_num_heads");
         if (n.inputs.size() > 12)
             return mfail(m->ctx, RTEN_ERR_UNSUPPORTED_VALUE, "GroupQueryAttention: quantization and Q/K norm inputs (12-15) are not supported");
         return RTEN_OK;
     }},
    {"MultiHeadAttention", MS, 0, 0b1, [](Runner& r, OpNode& o, rten_tensor* y) {
         rten_mha_params p;
         memset(&p, 0, sizeof(p));
         p.num_heads = (int32_t)o.n.attr_i("num_heads", 0);
         p.scale = o.n.attr_f("scale", 0.0f);
         p.mask_filter_value = o.n.attr_f("mask_filter_value", -10000.0f);
         p.unidirectional = (int32_t)o.n.attr_i("unidirectional", 0);
         rten_tensor pk{}, pv{};
         // new positions: key [B, L, H * D]; without key (packed QKV or self-attention on the query) the query's S
         const rten_tensor *q = r.T(o, 0), *k = r.T(o, 1);
         const int64_t L = k && k->ndim == 3 ? k->shape[1] : k ? -1 : (q->ndim >= 2 ? q->shape[1] : -1);
         const bool ik = L >= 0 && r.cache_in_place(o, 6, 1, L, &pk), iv = L >= 0 && r.cache_in_place(o, 7, 2, L, &pv);
         RTB_TRY(rten_b200_multi_head_attention(r.ctx, r.T(o, 0), r.T(o, 1), r.T(o, 2), r.T(o, 3), r.T(o, 4), r.T(o, 5), r.T(o, 6),
                                                r.T(o, 7), nullptr, nullptr, &p, y, r.wants(o, 1) ? &pk : nullptr, r.wants(o, 2) ? &pv : nullptr));
         r.set_present(o, 1, 6, ik, pk);
         r.set_present(o, 2, 7, iv, pv);
         return RTEN_OK;
     }, [](rten_model* m, onnx::Node& n) {  // src/op_registry/onnx_registry.rs:1495-1505, contrib.rs:302-315
         if (!n.attr("num_heads")) return mfail(m->ctx, RTEN_ERR_UNSUPPORTED_VALUE, "MultiHeadAttention: missing attribute num_heads");
         if (n.attr("scale") && !(n.attr_f("scale", 0.0f) > 0.0f))
             return mfail(m->ctx, RTEN_ERR_UNSUPPORTED_VALUE, "MultiHeadAttention: an explicit scale must be positive");
         for (size_t i = 8; i < n.inputs.size(); i++)
             if (!n.inputs[i].empty())
                 return mfail(m->ctx, RTEN_ERR_UNSUPPORTED_VALUE, "MultiHeadAttention: past_sequence_length and cache_indirection (inputs 8, 9) are not supported");
         if (n.outputs.size() > 3 && !n.outputs[3].empty())
             return mfail(m->ctx, RTEN_ERR_UNSUPPORTED_VALUE, "MultiHeadAttention: the qk output (3) is not supported");
         return RTEN_OK;
     }},
    {"GRU", ONNX, 0, 0b1, [](Runner& r, OpNode& o, rten_tensor* y) {
         const rten_rnn_params p = rnn_params(o.n);
         rten_tensor h{};
         RTB_TRY(rten_b200_gru(r.ctx, r.T(o, 0), r.T(o, 1), o.packed, r.T(o, 2), r.T(o, 3), r.T(o, 4), r.T(o, 5), &p,
                               r.wants(o, 0) ? y : nullptr, r.wants(o, 1) ? &h : nullptr));
         r.set_output(o, 1, h);
         return RTEN_OK;
     }, [](rten_model* m, onnx::Node& n) { return check_rnn_attrs(m->ctx, n, true); }, prepack_rnn},
    {"LSTM", ONNX, 0, 0b1, [](Runner& r, OpNode& o, rten_tensor* y) {
         const rten_rnn_params p = rnn_params(o.n);
         rten_tensor h{}, c{};
         RTB_TRY(rten_b200_lstm(r.ctx, r.T(o, 0), r.T(o, 1), o.packed, r.T(o, 2), r.T(o, 3), r.T(o, 4), r.T(o, 5), r.T(o, 6), nullptr, &p,
                                r.wants(o, 0) ? y : nullptr, r.wants(o, 1) ? &h : nullptr, r.wants(o, 2) ? &c : nullptr));
         r.set_output(o, 1, h);
         r.set_output(o, 2, c);
         return RTEN_OK;
     }, [](rten_model* m, onnx::Node& n) { return check_rnn_attrs(m->ctx, n, false); }, prepack_rnn},
    {"Where", ONNX, 0, 0b111, run_where},
    {"Equal", ONNX, 0, 0b11, run_compare<CMP_EQ>},
    {"Less", ONNX, 0, 0b11, run_compare<CMP_LT>},
    {"LessOrEqual", ONNX, 0, 0b11, run_compare<CMP_LE>},
    {"Greater", ONNX, 0, 0b11, run_compare<CMP_GT>},
    {"GreaterOrEqual", ONNX, 0, 0b11, run_compare<CMP_GE>},
    {"And", ONNX, 0, 0b11, [](Runner& r, OpNode& o, rten_tensor* y) { return rten_b200_and(r.ctx, r.T(o, 0), r.T(o, 1), y); }},
    {"Or", ONNX, 0, 0b11, [](Runner& r, OpNode& o, rten_tensor* y) { return rten_b200_or(r.ctx, r.T(o, 0), r.T(o, 1), y); }},
    {"Xor", ONNX, 0, 0b11, [](Runner& r, OpNode& o, rten_tensor* y) { return rten_b200_xor(r.ctx, r.T(o, 0), r.T(o, 1), y); }},
    {"Not", ONNX, 0, 0b1, [](Runner& r, OpNode& o, rten_tensor* y) { return rten_b200_not(r.ctx, r.T(o, 0), y); }},
    {"Expand", ONNX, 0, 0b11, run_expand},
    {"Slice", ONNX, 0, 0b1, run_slice},
    {"Split", ONNX, 0, 0b1, run_split},
    {"Range", ONNX, 0, 0b111, run_range},
    {"ConstantOfShape", ONNX, 0, 0b1, run_constant_of_shape},
    {"Trilu", ONNX, 0, 0b1, run_trilu},
    {"Constant", ONNX, 0, 0b1, nullptr},  // (becomes a constant value at load, not a node)
};

constexpr const OpDef* row(std::string_view name) {
    for (const OpDef& d : OPS)
        if (name == d.name) return &d;
    return nullptr;
}

// the operators the load-time passes look for
constexpr const OpDef *CONV = row("Conv"), *CONV_TRANSPOSE = row("ConvTranspose"), *CONCAT = row("Concat"), *SIGMOID = row("Sigmoid"),
                      *MUL = row("Mul"), *SILU = row("Silu"), *MATMUL = row("MatMul"), *ADD = row("Add"), *RESHAPE_OP = row("Reshape"),
                      *INSTANCE_NORM = row("InstanceNormalization"), *GROUP_NORM = row("GroupNorm"), *BATCH_NORM = row("BatchNormalization");
static_assert(CONV && CONV_TRANSPOSE && CONCAT && SIGMOID && MUL && SILU && MATMUL && ADD && RESHAPE_OP && INSTANCE_NORM && GROUP_NORM &&
                  BATCH_NORM,
              "a row the load looks for is missing");

// the decoded file as values and nodes: constants uploaded, every node checked against OPS
rten_status build_graph(rten_model* m, const onnx::Model& om) {
    rten_ctx* ctx = m->ctx;
    m->summary = onnx::summary_json(om);
    for (const onnx::Tensor& t : om.graph.initializers) RTB_TRY(upload_constant(m, t));
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
        // (domain, op_type) as the reference's registry looks it up (src/op_registry/onnx_registry.rs read_op)
        const OpDomain domain = n.domain == "com.microsoft" ? MS : ONNX;
        const OpDef* def = nullptr;
        for (const OpDef& d : OPS)
            if (n.op_type == d.name && (d.domains & domain)) def = &d;
        if (!def)
            return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "unsupported operator " + std::string(domain == MS ? "com.microsoft." : "") + n.op_type);
        if (n.op_type == "Constant") {
            const onnx::Attribute* a = n.attr("value");
            if (!a || !a->has_t || n.outputs.size() != 1) return mfail(ctx, RTEN_ERR_UNSUPPORTED_VALUE, "Constant without a tensor value");
            onnx::Tensor t = a->t;
            t.name = n.outputs[0];
            RTB_TRY(upload_constant(m, t));
            continue;
        }
        OpNode on;
        on.n = n;
        on.def = def;
        if (def->load) RTB_TRY(def->load(m, on.n));
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
    return RTEN_OK;
}

// ---- load-time passes (src/optimize.rs: the patterns the hot-path models contain)
// Who reads and who writes each value, over the nodes not absorbed: built when a fusion starts and again after each
// rewrite, never updated in place.
struct Uses {
    std::vector<int> uses;                  // the input slots that name the value, plus its places among the graph outputs
    std::vector<OpNode*> reader, producer;  // a node that reads it (the only one when uses == 1); the first that writes it
    explicit Uses(rten_model& m) : uses(m.values.size()), reader(m.values.size()), producer(m.values.size()) {
        for (OpNode& o : m.nodes) {
            if (!o.def) continue;
            for (int v : o.in)
                if (v >= 0) uses[(size_t)v]++, reader[(size_t)v] = &o;
            for (int v : o.out)
                if (v >= 0 && !producer[(size_t)v]) producer[(size_t)v] = &o;
        }
        for (int v : m.outputs) uses[(size_t)v]++;
    }
    // the node that reads `v` when that read is v's only use, else nullptr
    OpNode* sole_reader(int v) const { return v >= 0 && uses[(size_t)v] == 1 ? reader[(size_t)v] : nullptr; }
};

// One fusion: `fuse(node, uses)` on each node in order, true when it rewrote the graph.  It absorbs a node by clearing
// its `def`; absorbed nodes are skipped, and dropped at the end, the others keeping their order.
template <class Fuse>
void fuse_each(rten_model* m, Fuse fuse) {
    Uses u(*m);
    for (OpNode& o : m->nodes)
        if (o.def && fuse(o, u)) u = Uses(*m);
    m->nodes.erase(std::remove_if(m->nodes.begin(), m->nodes.end(), [](const OpNode& o) { return !o.def; }), m->nodes.end());
}

// what activation node `a` computes, as a fused epilogue takes it
rten_activation activation_of(const OpNode& a) {
    const bool hs = a.def->act == RTEN_ACT_HARD_SIGMOID;
    return {(int32_t)a.def->act, hs ? hard_sigmoid_alpha(a.n) : 0.0f, hs ? hard_sigmoid_beta(a.n) : 0.0f};
}

// SiluFusion (src/optimize/fusions.rs:567-588): Mul(x, Sigmoid(x)), either operand order, becomes Silu(x) in the Mul's
// place when the Sigmoid's output has no other use; Silu rounds once where the pair rounds twice, as the reference's
// Model::run does.  First: the Sigmoid and the Mul are two readers of a Conv's output, and GroupNormFusion takes the Silu.
void fuse_silu(rten_model* m) {
    fuse_each(m, [](OpNode& s, const Uses& u) {
        if (s.def != SIGMOID || s.in.size() != 1 || s.out.size() != 1) return false;
        OpNode* mul = u.sole_reader(s.out[0]);
        if (!mul || mul->def != MUL || mul->in.size() != 2 || mul->out.size() != 1) return false;
        const int x = s.in[0];
        if (!((mul->in[0] == s.out[0] && mul->in[1] == x) || (mul->in[1] == s.out[0] && mul->in[0] == x))) return false;
        mul->def = SILU;
        mul->n.op_type = SILU->name;
        mul->n.inputs = {s.n.inputs[0]};
        mul->n.attrs.clear();
        mul->in = {x};
        s.def = nullptr;
        return true;
    });
}

// GroupNormFusion: torch's export of nn.GroupNorm(G, C) -- Reshape(x, [0 | N, G, -1]) -> InstanceNormalization(
// scale [G], bias [G]) -> Reshape(to a constant 4-D shape) -> Mul(gamma [C, 1, 1]) -> Add(beta [C, 1, 1]), every
// intermediate with one reader -- and a following Relu / Sigmoid / Silu / HardSigmoid / HardSwish become one GroupNorm
// node in the last node's place: one pass over x instead of two copies, the norm and three elementwise launches.  The
// Reshape targets stay inputs, resolved for each run's x.  Only constant targets match, not one computed from Shape(x).
void fuse_group_norm(rten_model* m) {
    auto cval = [&](int vid) -> const ValueSlot* {
        return vid >= 0 && m->values[(size_t)vid].kind == V_CONST ? &m->values[(size_t)vid] : nullptr;
    };
    // a per-channel constant of C elements: [C], broadcast over the spatial axes, i.e. shape [.., C, 1, 1]
    auto per_channel = [&](int vid, int64_t* C) {
        const ValueSlot* v = cval(vid);
        if (!v || v->t.dtype != RTEN_F32 || v->t.ndim < 3 || v->t.ndim > 4) return false;
        const int nd = v->t.ndim;
        if (v->t.shape[nd - 1] != 1 || v->t.shape[nd - 2] != 1 || (nd == 4 && v->t.shape[0] != 1)) return false;
        *C = v->t.shape[nd - 3];
        return true;
    };
    fuse_each(m, [&](OpNode& r1, const Uses& u) {
        if (r1.def != RESHAPE_OP || r1.in.size() != 2 || r1.out.size() != 1 || r1.n.attr_i("allowzero", 0)) return false;
        const ValueSlot* t1 = cval(r1.in[1]);
        if (!t1 || !t1->has_host_ints || t1->host_ints.size() != 3 || t1->host_ints[0] < 0 || t1->host_ints[1] <= 0 ||
            t1->host_ints[2] != -1)
            return false;
        const int64_t G = t1->host_ints[1];
        OpNode* in = u.sole_reader(r1.out[0]);
        if (!in || in->def != INSTANCE_NORM || in->in.size() != 3 || in->in[0] != r1.out[0] || in->out.size() != 1) return false;
        const ValueSlot *sc = cval(in->in[1]), *bi = cval(in->in[2]);
        if (!sc || !bi || sc->t.ndim != 1 || bi->t.ndim != 1 || sc->t.shape[0] != G || bi->t.shape[0] != G) return false;
        OpNode* r2 = u.sole_reader(in->out[0]);
        if (!r2 || r2->def != RESHAPE_OP || r2->in.size() != 2 || r2->in[0] != in->out[0] || r2->out.size() != 1 ||
            r2->n.attr_i("allowzero", 0))
            return false;
        const ValueSlot* t2 = cval(r2->in[1]);
        if (!t2 || !t2->has_host_ints || t2->host_ints.size() != 4) return false;
        OpNode* mul = u.sole_reader(r2->out[0]);
        if (!mul || mul->def != MUL || mul->in.size() != 2 || mul->out.size() != 1) return false;
        const int gamma = mul->in[0] == r2->out[0] ? mul->in[1] : mul->in[0];
        int64_t C = 0, Cb = 0;
        if (gamma == r2->out[0] || !per_channel(gamma, &C) || C % G != 0) return false;
        OpNode* add = u.sole_reader(mul->out[0]);
        if (!add || add->def != ADD || add->in.size() != 2 || add->out.size() != 1) return false;
        const int beta = add->in[0] == mul->out[0] ? add->in[1] : add->in[0];
        if (beta == mul->out[0] || !per_channel(beta, &Cb) || Cb != C) return false;
        OpNode* last = add;
        OpNode* a = u.sole_reader(add->out[0]);
        if (a && a->def->act != RTEN_ACT_NONE && a->in.size() == 1 && a->out.size() == 1) last = a;
        in->def = GROUP_NORM;
        in->n.op_type = GROUP_NORM->name;
        in->in = {r1.in[0], in->in[1], in->in[2], gamma, beta, r1.in[1], r2->in[1]};
        in->out = last->out;
        if (last != add) in->activation = activation_of(*last);
        *last = *in;  // (every input exists by then)
        for (OpNode* o : {&r1, in, r2, mul, add})
            if (o != last) o->def = nullptr;
        return true;
    });
}

// The f32 elements of the constant `v`, copied back from the device
rten_status constant_floats(rten_model* m, int v, std::vector<float>* out) {
    const rten_tensor& t = m->values[(size_t)v].t;
    out->resize((size_t)numel(&t));
    if (!out->empty()) RTB_CUDA(m->ctx, cudaMemcpy(out->data(), t.data, out->size() * 4, cudaMemcpyDeviceToHost));
    return RTEN_OK;
}

// The constant `v` released: its device memory goes back to the pool and the value no longer exists.  Only for a
// constant nothing reads any more.
void release_constant(rten_model* m, int v) {
    ValueSlot& s = m->values[(size_t)v];
    m->const_allocs.erase(std::find(m->const_allocs.begin(), m->const_allocs.end(), s.t.data));
    pool_free(m->ctx, s.t.data);
    s.t.data = nullptr;
    s.kind = V_UNSET;
}

// Input `slot` of node o becomes a new f32 constant `name` of `dims` holding `data`.  The constant it replaces is
// released when o was its only reader (`uses`: its uses before the replacement).
rten_status replace_constant(rten_model* m, OpNode& o, size_t slot, int uses, const std::string& name, const std::vector<int64_t>& dims,
                             const std::vector<float>& data) {
    onnx::Tensor t;
    t.name = name;
    t.data_type = onnx::DT_FLOAT;
    t.dims = dims;
    t.data.resize(data.size() * 4);
    if (!data.empty()) memcpy(t.data.data(), data.data(), t.data.size());
    RTB_TRY(upload_constant(m, t));
    const int old = slot < o.in.size() ? o.in[slot] : -1;
    if (old >= 0 && uses == 1) release_constant(m, old);
    if (o.in.size() <= slot) o.in.resize(slot + 1, -1), o.n.inputs.resize(slot + 1);
    o.in[slot] = m->value_id(name);
    o.n.inputs[slot] = name;
    return RTEN_OK;
}

// Conv / ConvTranspose -> BatchNormalization, folded into the convolution at load when the BatchNormalization is the
// convolution's only reader, the convolution is f32 with a constant weight (and bias, when it has one) and no
// activation, and the four BatchNormalization parameters are constants of C_out elements.  On the host, in float32:
//   s[co] = scale[co] / sqrt(var[co] + epsilon)
//   w'[co, ..] = w[co, ..] * s[co]    (ConvTranspose: weight axis 1, co = g (C_out / G) + j)
//   b'[co] = fma(bias[co] - mean[co], s[co], beta[co])    (bias 0 without one): the operator applied to the bias
// The convolution takes the folded weights and the BatchNormalization's output, and the node launches nothing.  The
// replaced weights and the BatchNormalization's parameters are released where nothing else reads them.
rten_status fold_batch_norm(rten_model* m) {
    rten_status st = RTEN_OK;
    auto cval = [&](int vid, int64_t n) {
        if (vid < 0) return false;
        const ValueSlot& v = m->values[(size_t)vid];
        return v.kind == V_CONST && v.t.dtype == RTEN_F32 && v.t.ndim == 1 && v.t.shape[0] == n;
    };
    fuse_each(m, [&](OpNode& bn, const Uses& u) {
        if (st != RTEN_OK || bn.def != BATCH_NORM || bn.in.size() != 5) return false;
        for (size_t i = 1; i < bn.out.size(); i++)
            if (bn.out[i] >= 0) return false;
        const int x = bn.in[0];
        OpNode* c = x >= 0 ? u.producer[(size_t)x] : nullptr;
        if (!c || (c->def != CONV && c->def != CONV_TRANSPOSE) || c->out.size() != 1 || u.sole_reader(x) != &bn ||
            c->activation.kind != RTEN_ACT_NONE || c->in.size() < 2 || c->in[1] < 0)
            return false;
        const ValueSlot& wv = m->values[(size_t)c->in[1]];
        if (wv.kind != V_CONST || wv.t.dtype != RTEN_F32 || wv.t.ndim < 3) return false;
        const bool tr = c->def == CONV_TRANSPOSE;
        const int64_t G = c->n.attr_i("group", 1);
        if (G <= 0 || (tr && wv.t.shape[0] % G != 0)) return false;
        const int64_t co_n = tr ? wv.t.shape[1] * G : wv.t.shape[0];
        const int bias = c->in.size() > 2 ? c->in[2] : -1;
        if ((bias >= 0 && !cval(bias, co_n)) || !cval(bn.in[1], co_n) || !cval(bn.in[2], co_n) || !cval(bn.in[3], co_n) ||
            !cval(bn.in[4], co_n))
            return false;
        std::vector<float> w, b(co_n, 0.0f), scale, beta, mean, var;
        if ((st = constant_floats(m, c->in[1], &w)) != RTEN_OK || (bias >= 0 && (st = constant_floats(m, bias, &b)) != RTEN_OK) ||
            (st = constant_floats(m, bn.in[1], &scale)) != RTEN_OK || (st = constant_floats(m, bn.in[2], &beta)) != RTEN_OK ||
            (st = constant_floats(m, bn.in[3], &mean)) != RTEN_OK || (st = constant_floats(m, bn.in[4], &var)) != RTEN_OK)
            return false;
        const float eps = bn.n.attr_f("epsilon", 1e-5f);
        std::vector<float> s((size_t)co_n);
        for (int64_t k = 0; k < co_n; k++) {
            s[(size_t)k] = scale[(size_t)k] / std::sqrt(var[(size_t)k] + eps);
            b[(size_t)k] = std::fmaf(b[(size_t)k] - mean[(size_t)k], s[(size_t)k], beta[(size_t)k]);
        }
        // elements per output channel of one weight slice: Conv [C_out, C_in / G, k..], ConvTranspose [C_in, C_out / G, k..]
        const int64_t K = numel(&wv.t) / (wv.t.shape[0] * wv.t.shape[1]), cpg = wv.t.shape[1], cin_g = wv.t.shape[0] / G;
        for (size_t i = 0; i < w.size(); i++) {
            const int64_t co = tr ? (int64_t)i / (cpg * K) / cin_g * cpg + (int64_t)i / K % cpg : (int64_t)i / (cpg * K);
            w[i] = w[i] * s[(size_t)co];
        }
        const std::vector<int64_t> wdims(wv.t.shape, wv.t.shape + wv.t.ndim);
        const std::string tag = "/batch_norm_folded/" + m->values[(size_t)bn.out[0]].name;
        if ((st = replace_constant(m, *c, 1, u.uses[(size_t)c->in[1]], m->values[(size_t)c->in[1]].name + tag, wdims, w)) != RTEN_OK ||
            (st = replace_constant(m, *c, 2, bias >= 0 ? u.uses[(size_t)bias] : 0, "bias" + tag, {co_n}, b)) != RTEN_OK)
            return false;
        for (size_t i = 1; i < 5; i++)  // the parameters only this node read
            if (u.uses[(size_t)bn.in[i]] == 1) release_constant(m, bn.in[i]);
        c->out = bn.out;
        bn.def = nullptr;
        return true;
    });
    return st;
}

// Conv or BatchNormalization + activation -> the activation in the convolution epilogue / the normalization pass (Clip is
// not fused); MatMul + Add(constant vector over the last axis) -> FusedMatMul with a row bias (MatMulAddFusion).  The
// Conv / BatchNormalization / MatMul takes the absorbed node's output.
void fuse_into_producers(rten_model* m) {
    fuse_each(m, [&](OpNode& a, const Uses& u) {
        OpNode* b = a.out.size() == 1 ? u.sole_reader(a.out[0]) : nullptr;
        if (b && (a.def == CONV || a.def == BATCH_NORM) && a.activation.kind == RTEN_ACT_NONE && b->def->act != RTEN_ACT_NONE) {
            a.activation = activation_of(*b);
        } else if (b && a.def == MATMUL && b->def == ADD && a.bias_value < 0 && b->in.size() == 2) {
            const int other = b->in[0] == a.out[0] ? b->in[1] : b->in[0];
            const ValueSlot& bv = m->values[(size_t)other];
            const ValueSlot& wv = m->values[(size_t)a.in[1]];
            if (!(bv.kind == V_CONST && bv.t.dtype == RTEN_F32 && bv.t.ndim == 1 && wv.t.ndim >= 2 && wv.kind == V_CONST &&
                  bv.t.shape[0] == wv.t.shape[wv.t.ndim - 1]))
                return false;
            a.bias_value = other;
        } else {
            return false;
        }
        a.out = b->out;
        b->def = nullptr;
        return true;
    });
}

// Concat elision, decided once: which inputs of which channel Concat their producers write in place, reported as the
// summary's "concat_in_place" member.  `inputs`: the file's graph inputs, whose dims give their channel counts.
void plan_concat_elision(rten_model* m, const std::vector<onnx::ValueInfo>& inputs) {
    const Uses u(*m);
    std::map<std::string, std::vector<int64_t>> input_dims;
    for (const onnx::ValueInfo& vi : inputs) input_dims[vi.name] = vi.dims;
    // channels of a 4-D value as far as the file tells them, else -1
    std::function<int64_t(int, int)> channels = [&](int vid, int depth) -> int64_t {
        if (vid < 0 || depth > 64) return -1;
        const ValueSlot& v = m->values[(size_t)vid];
        if (v.kind == V_INPUT) {
            const std::vector<int64_t>& d = input_dims[v.name];
            return d.size() == 4 && d[1] > 0 ? d[1] : -1;
        }
        if (!u.producer[(size_t)vid]) return -1;
        const OpNode& p = *u.producer[(size_t)vid];
        auto weight = [&]() -> const rten_tensor* {
            if (p.in.size() < 2 || p.in[1] < 0 || m->values[(size_t)p.in[1]].kind != V_CONST) return nullptr;
            const rten_tensor& w = m->values[(size_t)p.in[1]].t;
            return w.ndim == 4 ? &w : nullptr;
        };
        if (p.def == CONV) return weight() ? weight()->shape[0] : -1;
        if (p.def == CONV_TRANSPOSE) return weight() ? weight()->shape[1] * p.n.attr_i("group", 1) : -1;
        // the pools and Resize / Upsample (the other Concat-slice writers) and the elementwise operators
        if (p.def->shape || (p.def->flags & IN_PLACE)) return channels(p.in[0], depth + 1);
        if (p.def == CONCAT && p.n.attr_i("axis", 0) == 1) {
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
        if (c.def != CONCAT || c.n.attr_i("axis", 0) != 1 || c.out.size() != 1 || c.out[0] < 0 || u.uses[(size_t)c.out[0]] < 1) continue;
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
            OpNode& p = *u.producer[(size_t)vid];
            if (!p.def->shape || p.out.size() != 1 || p.cat_node >= 0) continue;
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

// constant weights prepacked once (`Operator::prepack`, src/graph.rs:488-565)
rten_status prepack_weights(rten_model* m) {
    for (OpNode& o : m->nodes) {
        const int w = o.in.size() >= 2 ? o.in[1] : -1;
        if (o.def->prepack && w >= 0 && m->values[(size_t)w].kind == V_CONST) RTB_TRY(o.def->prepack(m->ctx, o, m->values[(size_t)w].t));
    }
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
    RTB_TRY(build_graph(m.get(), om));
    fuse_silu(m.get());
    if (!getenv("RTEN_B200_NO_GROUP_NORM_FUSION")) fuse_group_norm(m.get());
    RTB_TRY(fold_batch_norm(m.get()));
    fuse_into_producers(m.get());
    if (!getenv("RTEN_B200_NO_CONCAT_ELISION")) plan_concat_elision(m.get(), om.graph.inputs);
    RTB_TRY(prepack_weights(m.get()));
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

rten_status rten_b200_model_run(rten_model* m, int32_t n_inputs, const char* const* input_names, const rten_tensor* inputs,
                                int32_t n_outputs, const char* const* output_names, rten_tensor* outputs) {
    return rten_b200_model_run_ex(m, n_inputs, input_names, inputs, nullptr, n_outputs, output_names, outputs, nullptr);
}

// A writable input's strides are those of a dense tensor whose grow axis has `capacity` positions
static bool dense_with_capacity(const rten_tensor& t, int grow_axis, int64_t capacity) {
    int64_t st = 1;
    for (int i = t.ndim - 1; i >= 0; i--) {
        const int64_t n = i == grow_axis ? capacity : t.shape[i];
        if (n != 1 && t.strides[i] != st) return false;
        st *= n;
    }
    return true;
}

rten_status rten_b200_model_run_ex(rten_model* m, int32_t n_inputs, const char* const* input_names, const rten_tensor* inputs,
                                   const rten_model_input_opts* opts, int32_t n_outputs, const char* const* output_names,
                                   rten_tensor* outputs, int32_t* output_alias) {
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
            v.writable = false;
            v.grow_axis = -1;
            v.capacity = 0;
            v.input_index = -1;
            v.alias_of = -1;
            if (v.kind == V_TEMP) {
                v.t.data = nullptr;
                v.has_host_ints = false;
                v.host_ints.clear();
            }
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
        if (opts && opts[i].writable) {
            const rten_model_input_opts& op = opts[i];
            const rten_tensor& t = inputs[i];
            if (t.device < 0)
                return cleanup(mfail(ctx, RTEN_ERR_INVALID_VALUE, std::string("writable input '") + input_names[i] + "' must be device-resident"));
            if (op.grow_axis < -1 || op.grow_axis >= t.ndim || (op.grow_axis >= 0 && op.capacity < t.shape[op.grow_axis]) ||
                !dense_with_capacity(t, op.grow_axis, op.grow_axis >= 0 ? op.capacity : 0))
                return cleanup(mfail(ctx, RTEN_ERR_INVALID_VALUE, std::string("writable input '") + input_names[i] +
                                                                      "': strides must be dense with capacity >= shape on grow_axis"));
            v.writable = true;
            v.grow_axis = op.grow_axis;
            v.capacity = op.grow_axis >= 0 ? op.capacity : 0;
        }
        v.input_index = i;
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
        for (int i : o.in) r.consumed(i);
    }
    // hand the requested outputs over: owned buffers move to the caller; a present cache written into a writable input is
    // returned as that view (output_alias names the input); other views / constants / inputs are copied
    for (int32_t i = 0; i < n_outputs; i++) {
        ValueSlot& v = m->values[(size_t)want[(size_t)i]];
        if (!v.live && v.kind != V_CONST) return cleanup(mfail(ctx, RTEN_ERR_INVALID_VALUE, "requested output '" + v.name + "' was not computed"));
        if (output_alias) output_alias[i] = -1;
        if (v.alias_of >= 0 && output_alias) {
            outputs[i] = v.t;
            output_alias[i] = v.alias_of;
            continue;
        }
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
            c.device = ctx->device;  // (a host value is handed over in HBM like every other output)
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

}  // extern "C"
