// ONNX wire-format decoder (host code only; compiled by nvcc with the rest of the library).  See onnx_reader.h.
// Field numbers follow onnx.proto3 as restated in rten-onnx/src/onnx.rs.
#include "onnx_reader.h"

#include <cstring>
#include <sstream>

namespace rtb {
namespace onnx {

namespace {

struct Reader {
    const uint8_t* p;
    const uint8_t* end;
    bool ok = true;

    bool done() const { return p >= end; }
    uint64_t varint() {
        uint64_t v = 0;
        int shift = 0;
        while (p < end && shift < 64) {
            const uint8_t c = *p++;
            v |= (uint64_t)(c & 0x7F) << shift;
            if (!(c & 0x80)) return v;
            shift += 7;
        }
        ok = false;
        return 0;
    }
    // next field: number, wire type; for length-delimited fields `sub` spans the payload
    bool next(uint32_t* field, uint32_t* wt, uint64_t* val, Reader* sub) {
        if (done() || !ok) return false;
        const uint64_t key = varint();
        if (!ok) return false;
        *field = (uint32_t)(key >> 3);
        *wt = (uint32_t)(key & 7);
        switch (*wt) {
            case 0: *val = varint(); break;
            case 1:
                if (end - p < 8) return ok = false;
                memcpy(val, p, 8);
                p += 8;
                break;
            case 2: {
                const uint64_t n = varint();
                if (!ok || n > (uint64_t)(end - p)) return ok = false;
                sub->p = p;
                sub->end = p + n;
                sub->ok = true;
                p += n;
                break;
            }
            case 5: {
                if (end - p < 4) return ok = false;
                uint32_t v32;
                memcpy(&v32, p, 4);
                *val = v32;
                p += 4;
                break;
            }
            default: return ok = false;  // groups are not used by ONNX
        }
        return ok;
    }
    std::string str() const { return std::string(reinterpret_cast<const char*>(p), (size_t)(end - p)); }
};

// repeated scalar field: packed (wire type 2) or one value per key
template <typename T, typename F>
void repeated(uint32_t wt, uint64_t val, Reader sub, std::vector<T>* out, F conv) {
    if (wt == 2) {
        while (!sub.done() && sub.ok) out->push_back(conv(sub.varint()));
    } else {
        out->push_back(conv(val));
    }
}

int elem_size(int32_t dt) {
    switch (dt) {
        case DT_FLOAT: case DT_INT32: return 4;
        case DT_INT64: return 8;
        case DT_UINT8: case DT_INT8: case DT_BOOL: return 1;
        default: return 0;
    }
}

bool decode_tensor(Reader r, Tensor* t, std::string* err) {
    std::vector<float> fdata;
    std::vector<int64_t> i32data, i64data;
    uint32_t f, wt;
    uint64_t v;
    Reader sub{nullptr, nullptr};
    bool has_raw = false;
    while (r.next(&f, &wt, &v, &sub)) {
        switch (f) {
            case 1: repeated<int64_t>(wt, v, sub, &t->dims, [](uint64_t x) { return (int64_t)x; }); break;
            case 2: t->data_type = (int32_t)v; break;
            case 4:  // float_data: packed fixed32 or single fixed32
                if (wt == 2) {
                    const size_t n = (size_t)(sub.end - sub.p) / 4;
                    const size_t o = fdata.size();
                    fdata.resize(o + n);
                    memcpy(fdata.data() + o, sub.p, n * 4);
                } else {
                    float x;
                    const uint32_t b = (uint32_t)v;
                    memcpy(&x, &b, 4);
                    fdata.push_back(x);
                }
                break;
            case 5: repeated<int64_t>(wt, v, sub, &i32data, [](uint64_t x) { return (int64_t)(int32_t)(uint32_t)x; }); break;
            case 7: repeated<int64_t>(wt, v, sub, &i64data, [](uint64_t x) { return (int64_t)x; }); break;
            case 8: t->name = sub.str(); break;
            case 9:
                t->data.assign(sub.p, sub.end);
                has_raw = true;
                break;
            case 14: t->external = (v == 1); break;
            default: break;  // doc_string, segment, external_data, ...: skipped
        }
    }
    if (!r.ok) {
        *err = "malformed TensorProto";
        return false;
    }
    const int es = elem_size(t->data_type);
    if (!has_raw && es) {
        const int64_t n = t->numel();
        t->data.resize((size_t)n * es);
        if (t->data_type == DT_FLOAT && (int64_t)fdata.size() == n) {
            memcpy(t->data.data(), fdata.data(), (size_t)n * 4);
        } else if (t->data_type == DT_INT64 && (int64_t)i64data.size() == n) {
            memcpy(t->data.data(), i64data.data(), (size_t)n * 8);
        } else if ((int64_t)i32data.size() == n && t->data_type != DT_FLOAT && t->data_type != DT_INT64) {
            for (int64_t i = 0; i < n; i++) {  // int32_data carries INT32 / INT8 / UINT8 / BOOL elements
                if (es == 4) {
                    const int32_t x = (int32_t)i32data[(size_t)i];
                    memcpy(t->data.data() + 4 * i, &x, 4);
                } else {
                    t->data[(size_t)i] = (uint8_t)i32data[(size_t)i];
                }
            }
        } else if (!t->external && n != 0) {
            *err = "TensorProto '" + t->name + "' has no data for its shape";
            return false;
        }
    }
    if (has_raw && es && !t->external && (int64_t)t->data.size() != t->numel() * es) {
        *err = "TensorProto '" + t->name + "': raw_data size does not match its shape";
        return false;
    }
    return true;
}

bool decode_attribute(Reader r, Attribute* a, std::string* err) {
    uint32_t f, wt;
    uint64_t v;
    Reader sub{nullptr, nullptr};
    while (r.next(&f, &wt, &v, &sub)) {
        switch (f) {
            case 1: a->name = sub.str(); break;
            case 2: {
                const uint32_t b = (uint32_t)v;
                memcpy(&a->f, &b, 4);
                a->has_f = true;
                break;
            }
            case 3:
                a->i = (int64_t)v;
                a->has_i = true;
                break;
            case 4: a->s = sub.str(); break;
            case 5:
                if (!decode_tensor(sub, &a->t, err)) return false;
                a->has_t = true;
                break;
            case 7:
                if (wt == 2) {
                    const size_t n = (size_t)(sub.end - sub.p) / 4;
                    const size_t o = a->floats.size();
                    a->floats.resize(o + n);
                    memcpy(a->floats.data() + o, sub.p, n * 4);
                } else {
                    float x;
                    const uint32_t b = (uint32_t)v;
                    memcpy(&x, &b, 4);
                    a->floats.push_back(x);
                }
                break;
            case 8: repeated<int64_t>(wt, v, sub, &a->ints, [](uint64_t x) { return (int64_t)x; }); break;
            case 9:  // strings: one length-delimited entry per string
                if (wt != 2) {
                    *err = "malformed AttributeProto";
                    return false;
                }
                a->strings.push_back(sub.str());
                break;
            case 20: a->type = (int32_t)v; break;
            default: break;
        }
    }
    if (!r.ok) *err = "malformed AttributeProto";
    return r.ok;
}

bool decode_node(Reader r, Node* n, std::string* err) {
    uint32_t f, wt;
    uint64_t v;
    Reader sub{nullptr, nullptr};
    while (r.next(&f, &wt, &v, &sub)) {
        switch (f) {
            case 1: n->inputs.push_back(sub.str()); break;
            case 2: n->outputs.push_back(sub.str()); break;
            case 3: n->name = sub.str(); break;
            case 4: n->op_type = sub.str(); break;
            case 5: {
                Attribute a;
                if (!decode_attribute(sub, &a, err)) return false;
                n->attrs.push_back(std::move(a));
                break;
            }
            case 7: n->domain = sub.str(); break;
            default: break;
        }
    }
    if (!r.ok) *err = "malformed NodeProto";
    return r.ok;
}

// ValueInfoProto { name = 1, type = 2 { tensor_type = 1 { elem_type = 1, shape = 2 { dim = 1 { dim_value = 1 | dim_param = 2 } } } } }
bool decode_value_info(Reader r, ValueInfo* vi) {
    uint32_t f, wt;
    uint64_t v;
    Reader sub{nullptr, nullptr};
    while (r.next(&f, &wt, &v, &sub)) {
        if (f == 1) {
            vi->name = sub.str();
        } else if (f == 2 && wt == 2) {
            Reader ty = sub, s2{nullptr, nullptr};
            while (ty.next(&f, &wt, &v, &s2)) {
                if (f != 1 || wt != 2) continue;  // tensor_type
                Reader tt = s2, s3{nullptr, nullptr};
                while (tt.next(&f, &wt, &v, &s3)) {
                    if (f == 1) {
                        vi->elem_type = (int32_t)v;
                    } else if (f == 2 && wt == 2) {
                        Reader sh = s3, s4{nullptr, nullptr};
                        while (sh.next(&f, &wt, &v, &s4)) {
                            if (f != 1 || wt != 2) continue;  // dim
                            Reader dm = s4, s5{nullptr, nullptr};
                            int64_t dv = -1;
                            while (dm.next(&f, &wt, &v, &s5))
                                if (f == 1) dv = (int64_t)v;
                            vi->dims.push_back(dv);
                        }
                    }
                }
            }
        }
    }
    return r.ok;
}

bool decode_graph(Reader r, Graph* g, std::string* err) {
    uint32_t f, wt;
    uint64_t v;
    Reader sub{nullptr, nullptr};
    while (r.next(&f, &wt, &v, &sub)) {
        switch (f) {
            case 1: {
                Node n;
                if (!decode_node(sub, &n, err)) return false;
                g->nodes.push_back(std::move(n));
                break;
            }
            case 2: g->name = sub.str(); break;
            case 5: {
                Tensor t;
                if (!decode_tensor(sub, &t, err)) return false;
                g->initializers.push_back(std::move(t));
                break;
            }
            case 11: case 12: {
                ValueInfo vi;
                if (!decode_value_info(sub, &vi)) {
                    *err = "malformed ValueInfoProto";
                    return false;
                }
                (f == 11 ? g->inputs : g->outputs).push_back(std::move(vi));
                break;
            }
            default: break;
        }
    }
    if (!r.ok) *err = "malformed GraphProto";
    return r.ok;
}

void json_str(std::ostringstream& o, const std::string& s) {
    o << '"';
    for (char c : s) {
        if (c == '"' || c == '\\')
            o << '\\' << c;
        else if ((unsigned char)c < 0x20)
            o << ' ';
        else
            o << c;
    }
    o << '"';
}

}  // namespace

bool decode_model(const uint8_t* bytes, size_t len, Model* out, std::string* err) {
    Reader r{bytes, bytes + len};
    uint32_t f, wt;
    uint64_t v;
    Reader sub{nullptr, nullptr};
    while (r.next(&f, &wt, &v, &sub)) {
        switch (f) {
            case 1: out->ir_version = (int64_t)v; break;
            case 7:
                if (wt != 2 || !decode_graph(sub, &out->graph, err)) {
                    if (err->empty()) *err = "malformed ModelProto";
                    return false;
                }
                out->has_graph = true;
                break;
            case 8: {  // opset_import { domain = 1, version = 2 }
                if (wt != 2) break;
                Reader os = sub, s2{nullptr, nullptr};
                std::string domain;
                int64_t version = 0;
                while (os.next(&f, &wt, &v, &s2)) {
                    if (f == 1) domain = s2.str();
                    if (f == 2) version = (int64_t)v;
                }
                out->opset[domain] = version;
                break;
            }
            default: break;
        }
    }
    if (!r.ok) {
        *err = "malformed ModelProto";
        return false;
    }
    return true;
}

std::string summary_json(const Model& m) {
    std::ostringstream o;
    o << "{\"ir_version\": " << m.ir_version << ", \"has_graph\": " << (m.has_graph ? "true" : "false") << ", \"opset\": {";
    bool first = true;
    for (const auto& kv : m.opset) {
        if (!first) o << ", ";
        first = false;
        json_str(o, kv.first);
        o << ": " << kv.second;
    }
    o << "}, \"nodes\": [";
    for (size_t i = 0; i < m.graph.nodes.size(); i++) {
        const Node& n = m.graph.nodes[i];
        if (i) o << ", ";
        o << "{\"op\": ";
        json_str(o, n.op_type);
        o << ", \"inputs\": [";
        for (size_t k = 0; k < n.inputs.size(); k++) {
            if (k) o << ", ";
            json_str(o, n.inputs[k]);
        }
        o << "], \"outputs\": [";
        for (size_t k = 0; k < n.outputs.size(); k++) {
            if (k) o << ", ";
            json_str(o, n.outputs[k]);
        }
        o << "], \"attrs\": [";
        for (size_t k = 0; k < n.attrs.size(); k++) {
            if (k) o << ", ";
            json_str(o, n.attrs[k].name);
        }
        o << "]";
        // the values of STRINGS attributes (e.g. an RNN's activations), by attribute name
        bool any = false;
        for (const Attribute& a : n.attrs) {
            if (a.strings.empty()) continue;
            o << (any ? ", " : ", \"strings\": {");
            any = true;
            json_str(o, a.name);
            o << ": [";
            for (size_t k = 0; k < a.strings.size(); k++) {
                if (k) o << ", ";
                json_str(o, a.strings[k]);
            }
            o << "]";
        }
        o << (any ? "}}" : "}");
    }
    o << "], \"initializers\": [";
    for (size_t i = 0; i < m.graph.initializers.size(); i++) {
        const Tensor& t = m.graph.initializers[i];
        if (i) o << ", ";
        o << "{\"name\": ";
        json_str(o, t.name);
        o << ", \"data_type\": " << t.data_type << ", \"dims\": [";
        for (size_t k = 0; k < t.dims.size(); k++) o << (k ? ", " : "") << t.dims[k];
        o << "], \"bytes\": " << t.data.size() << "}";
    }
    auto vis = [&](const char* key, const std::vector<ValueInfo>& v) {
        o << ", \"" << key << "\": [";
        for (size_t i = 0; i < v.size(); i++) {
            if (i) o << ", ";
            o << "{\"name\": ";
            json_str(o, v[i].name);
            o << ", \"elem_type\": " << v[i].elem_type << ", \"dims\": [";
            for (size_t k = 0; k < v[i].dims.size(); k++) o << (k ? ", " : "") << v[i].dims[k];
            o << "]}";
        }
        o << "]";
    };
    o << "]";
    vis("inputs", m.graph.inputs);
    vis("outputs", m.graph.outputs);
    o << "}";
    return o.str();
}

}  // namespace onnx
}  // namespace rtb
