// Minimal ONNX reader: the subset of the protobuf schema the hot-path models use, decoded straight from the wire format
// (no protobuf library), like the reference's own hand-written decoder (rten-onnx/src/onnx.rs:17-700,
// rten-onnx/src/protobuf.rs).  Host-only: usable without a GPU.
#pragma once
#include <cstddef>
#include <cstdint>
#include <map>
#include <string>
#include <vector>

namespace rtb {
namespace onnx {

// TensorProto.DataType values that occur on the path (rten-onnx/src/onnx.rs:271-338)
enum DataType : int32_t { DT_UNDEFINED = 0, DT_FLOAT = 1, DT_UINT8 = 2, DT_INT8 = 3, DT_INT32 = 6, DT_INT64 = 7, DT_BOOL = 9 };

struct Tensor {
    std::string name;
    int32_t data_type = DT_UNDEFINED;
    std::vector<int64_t> dims;
    std::vector<uint8_t> data;  // little-endian elements of `data_type`, whatever field the file used
    bool external = false;      // data_location = EXTERNAL (not loaded)
    int64_t numel() const {
        int64_t n = 1;
        for (int64_t d : dims) n *= d;
        return n;
    }
};

// AttributeProto (rten-onnx/src/onnx.rs:30-103)
struct Attribute {
    std::string name;
    int32_t type = 0;  // 1 FLOAT, 2 INT, 3 STRING, 4 TENSOR, 6 FLOATS, 7 INTS, 8 STRINGS
    float f = 0.0f;
    int64_t i = 0;
    std::string s;
    std::vector<float> floats;
    std::vector<int64_t> ints;
    std::vector<std::string> strings;
    Tensor t;
    bool has_f = false, has_i = false, has_t = false;
};

struct Node {
    std::string name, op_type, domain;
    std::vector<std::string> inputs, outputs;
    std::vector<Attribute> attrs;
    const Attribute* attr(const char* n) const {
        for (const Attribute& a : attrs)
            if (a.name == n) return &a;
        return nullptr;
    }
    int64_t attr_i(const char* n, int64_t dflt) const {
        const Attribute* a = attr(n);
        return (a && a->has_i) ? a->i : dflt;
    }
    float attr_f(const char* n, float dflt) const {
        const Attribute* a = attr(n);
        return (a && a->has_f) ? a->f : dflt;
    }
    std::vector<int64_t> attr_ints(const char* n) const {
        const Attribute* a = attr(n);
        return a ? a->ints : std::vector<int64_t>();
    }
};

struct ValueInfo {
    std::string name;
    int32_t elem_type = 0;
    std::vector<int64_t> dims;  // -1 for symbolic / unknown
};

struct Graph {
    std::string name;
    std::vector<Node> nodes;
    std::vector<Tensor> initializers;
    std::vector<ValueInfo> inputs, outputs;
};

struct Model {
    int64_t ir_version = -1;
    std::map<std::string, int64_t> opset;  // domain ("" = default) -> version
    bool has_graph = false;
    Graph graph;
};

// Decodes `len` bytes; false (with `err`) on malformed input.  An empty buffer decodes to a default Model without a
// graph, as the reference's decoder does (rten-onnx/src/onnx.rs:798-804).
bool decode_model(const uint8_t* bytes, size_t len, Model* out, std::string* err);

// JSON description of the decoded structure (operators, initialisers, inputs / outputs), for tests and tooling.
std::string summary_json(const Model& m);

}  // namespace onnx
}  // namespace rtb
