// Graph: *.anakin.bin reader / writer (hand-written proto3 wire codec -- no protobuf in this
// image) and the fusion / ordering passes of Graph::Optimize.
//   file format  reference framework/model_parser/proto/{graph,node,tensor,operator}.proto
//   load         reference framework/model_parser/parser/parser.cpp:67-237, model_io.cpp:9-260
//   Optimize     reference framework/graph/graph.cpp:350-472,588-804
#include "graph.h"

#include <stdlib.h>

#include "../image_desc.h"

#include <algorithm>
#include <fstream>
#include <functional>
#include <set>

namespace anakin {
namespace graph {

using saber::Shape;

// ------------------------------------------------------------------ proto3 wire helpers
namespace {

enum DateTypeProto { P_STR = 0, P_INT8 = 2, P_INT32 = 4, P_FLOAT16 = 8, P_FLOAT = 13, P_DOUBLE = 14,
                     P_BOOLEN = 20, P_CACHE_LIST = 30, P_TENSOR = 31 };

struct Reader {
    const uint8_t* p;
    const uint8_t* end;
    bool ok = true;
    Reader(const void* b, size_t n) : p(static_cast<const uint8_t*>(b)), end(p + n) {}
    bool done() const { return p >= end || !ok; }
    uint64_t varint() {
        uint64_t r = 0;
        int shift = 0;
        while (p < end) {
            uint8_t b = *p++;
            r |= static_cast<uint64_t>(b & 0x7F) << shift;
            if (!(b & 0x80)) return r;
            shift += 7;
            if (shift > 63) break;
        }
        ok = false;
        return 0;
    }
    // reads a field header; for wire type 2 returns the sub-range in (sub)
    bool next(int& field, int& wt, uint64_t& val, Reader& sub) {
        if (done()) return false;
        uint64_t key = varint();
        field = static_cast<int>(key >> 3);
        wt = static_cast<int>(key & 7);
        if (wt == 0) {
            val = varint();
        } else if (wt == 2) {
            uint64_t len = varint();
            if (!ok || len > static_cast<uint64_t>(end - p)) { ok = false; return false; }
            sub = Reader(p, static_cast<size_t>(len));
            p += len;
        } else if (wt == 5) {
            if (end - p < 4) { ok = false; return false; }
            uint32_t v; memcpy(&v, p, 4); p += 4; val = v;
        } else if (wt == 1) {
            if (end - p < 8) { ok = false; return false; }
            memcpy(&val, p, 8); p += 8;
        } else {
            ok = false;
            return false;
        }
        return ok;
    }
    std::string str() const { return std::string(reinterpret_cast<const char*>(p), static_cast<size_t>(end - p)); }
};

struct Writer {
    std::string buf;
    void varint(uint64_t v) {
        while (v >= 0x80) { buf.push_back(static_cast<char>((v & 0x7F) | 0x80)); v >>= 7; }
        buf.push_back(static_cast<char>(v));
    }
    void tag(int field, int wt) { varint((static_cast<uint64_t>(field) << 3) | wt); }
    void f_varint(int field, uint64_t v) { tag(field, 0); varint(v); }
    void f_bytes(int field, const std::string& s) { tag(field, 2); varint(s.size()); buf += s; }
    void f_bytes(int field, const void* d, size_t n) { tag(field, 2); varint(n); buf.append(static_cast<const char*>(d), n); }
    void f_float(int field, float f) { tag(field, 5); buf.append(reinterpret_cast<const char*>(&f), 4); }
};

struct CacheData {
    std::vector<std::string> s;
    std::vector<int> i;
    std::vector<float> f;
    std::vector<bool> b;
    std::string c;          // CacheDate.c: int8 payload (tensor.proto field 8)
    int type = 0;
    long long size = -1;    // CacheDate.size (field 7); -1 = absent
};

CacheData read_cache(Reader r) {
    CacheData c;
    int field, wt; uint64_t v; Reader sub(nullptr, 0);
    while (r.next(field, wt, v, sub)) {
        switch (field) {
            case 1: c.s.push_back(sub.str()); break;
            case 2:
                if (wt == 2) { while (!sub.done()) c.i.push_back(static_cast<int>(static_cast<int64_t>(sub.varint()))); }
                else c.i.push_back(static_cast<int>(static_cast<int64_t>(v)));
                break;
            case 3:
                if (wt == 2) {
                    size_t n = static_cast<size_t>(sub.end - sub.p) / 4;
                    size_t o = c.f.size();
                    c.f.resize(o + n);
                    memcpy(c.f.data() + o, sub.p, n * 4);
                } else { uint32_t u = static_cast<uint32_t>(v); float f; memcpy(&f, &u, 4); c.f.push_back(f); }
                break;
            case 4:
                if (wt == 2) { while (!sub.done()) c.b.push_back(sub.varint() != 0); }
                else c.b.push_back(v != 0);
                break;
            case 8: c.c = sub.str(); break;
            case 6: c.type = static_cast<int>(v); break;
            case 7: c.size = static_cast<long long>(v); break;
            default: break;
        }
    }
    return c;
}

std::vector<int> read_shape(Reader r) {
    std::vector<int> dims;
    int field, wt; uint64_t v; Reader sub(nullptr, 0);
    while (r.next(field, wt, v, sub)) {
        if (field != 3 || wt != 2) continue;
        int f2, w2; uint64_t v2; Reader s2(nullptr, 0);
        while (sub.next(f2, w2, v2, s2)) {
            if (f2 == 1) {
                if (w2 == 2) { while (!s2.done()) dims.push_back(static_cast<int>(s2.varint())); }
                else dims.push_back(static_cast<int>(v2));
            }
        }
    }
    return dims;
}

struct TensorData {
    std::vector<int> shape, valid_shape;
    std::vector<float> data, scale;
    std::string q8;          // int8 codes when data_type == P_INT8
    int data_type = P_FLOAT;
    long long data_size = -1;
    bool shared = false;
    std::string share_from;
};

TensorData read_tensor(Reader r) {
    TensorData t;
    int field, wt; uint64_t v; Reader sub(nullptr, 0);
    while (r.next(field, wt, v, sub)) {
        switch (field) {
            case 2: t.shared = v != 0; break;
            case 3: t.share_from = sub.str(); break;
            case 8: t.shape = read_shape(sub); break;
            case 9: t.valid_shape = read_shape(sub); break;
            case 10: {
                CacheData c = read_cache(sub);
                t.data = std::move(c.f);
                t.q8 = std::move(c.c);
                // proto3 drops a zero enum: an absent type with int8 bytes present still means INT8
                t.data_type = c.type == P_INT8 || (c.type == 0 && !t.q8.empty() && t.data.empty()) ? P_INT8 : P_FLOAT;
                t.data_size = c.size;
            } break;
            case 11: t.scale = read_cache(sub).f; break;
            default: break;
        }
    }
    return t;
}

// model_io.cpp:152-216: a FLOAT tensor becomes an fp32 block, an INT8 tensor an int8 block carrying its
// per-output-channel scales; the real shape allocates, a present valid_shape re-shapes. A payload that does not
// fill the shape is an error here (the reference would read past the repeated field and abort).
PBlockPtr make_block(const TensorData& t, std::string* err) {
    PBlockPtr b = std::make_shared<PBlock>();
    std::vector<int> sh = t.shape;
    while (sh.size() < 4) sh.insert(sh.begin(), 1);
    const bool q8 = t.data_type == P_INT8;
    b->h.re_alloc(Shape(sh, saber::Layout_NCHW), q8 ? saber::AK_INT8 : saber::AK_FLOAT);
    const size_t cnt = static_cast<size_t>(b->h.valid_size());
    const size_t have = q8 ? t.q8.size() : t.data.size();
    if (have != cnt) {
        if (err) *err = "tensor payload holds " + std::to_string(have) + " elements, shape needs " + std::to_string(cnt);
        return nullptr;
    }
    if (cnt) {
        if (q8) memcpy(b->h.mutable_data(), t.q8.data(), cnt);
        else memcpy(b->h.mutable_data(), t.data.data(), cnt * sizeof(float));
    }
    b->h.set_scale(t.scale);
    if (t.valid_shape.size() == 4 && t.valid_shape != sh) b->h.set_shape(Shape(t.valid_shape, saber::Layout_NCHW));
    return b;
}

// `share_from` receives the owner node's name when the value is a shared tensor (TensorProto.shared): the caller
// points the attribute at that node's block once every node is parsed (model_io.cpp:147-151).
bool read_value(Reader r, AttrValue& out, std::string* share_from, std::string* err) {
    int type = P_STR;
    std::string s; int i = 0; float f = 0.f; bool b = false;
    CacheData cache; TensorData tensor; bool has_tensor = false;
    int field, wt; uint64_t v; Reader sub(nullptr, 0);
    while (r.next(field, wt, v, sub)) {
        switch (field) {
            case 1: s = sub.str(); break;
            case 2: i = static_cast<int>(static_cast<int64_t>(v)); break;
            case 3: { uint32_t u = static_cast<uint32_t>(v); memcpy(&f, &u, 4); } break;
            case 4: b = v != 0; break;
            case 8: cache = read_cache(sub); break;
            case 10: tensor = read_tensor(sub); has_tensor = true; break;
            case 14: type = static_cast<int>(v); break;
            default: break;
        }
    }
    switch (type) {
        case P_STR: out = s; return true;
        case P_INT32: out = i; return true;
        case P_FLOAT: case P_DOUBLE: out = f; return true;
        case P_BOOLEN: out = b; return true;
        case P_CACHE_LIST:
            switch (cache.type) {
                case P_FLOAT: out = cache.f; return true;
                case P_BOOLEN: out = cache.b; return true;
                case P_STR: out = cache.s; return true;
                default: out = cache.i; return true;
            }
        case P_TENSOR:
            if (!has_tensor) return false;
            if (tensor.shared) {
                if (tensor.share_from.empty()) { if (err) *err = "shared tensor without share_from"; return false; }
                if (share_from) *share_from = tensor.share_from;
                out = PBlockPtr();
                return true;
            }
            {
                PBlockPtr blk = make_block(tensor, err);
                if (!blk) return false;
                out = blk;
            }
            return true;
        default: return false;
    }
}

void write_cache_floats(Writer& w, const float* d, size_t n) {
    if (n) w.f_bytes(3, d, n * 4);
    w.f_varint(6, P_FLOAT);
    if (n) w.f_varint(7, n);
}

std::string enc_shape(const std::vector<int>& dims) {
    Writer vals;
    for (int d : dims) vals.varint(static_cast<uint64_t>(d));
    Writer dim;
    dim.f_bytes(1, vals.buf);
    dim.f_varint(2, dims.size());
    Writer sh;
    sh.f_bytes(3, dim.buf);
    return sh.buf;
}

std::string enc_value(const AttrValue& v, const std::string* share_from = nullptr) {
    Writer w;
    if (auto p = std::get_if<std::string>(&v)) {
        w.f_bytes(1, *p);
    } else if (auto p = std::get_if<int>(&v)) {
        if (*p) w.f_varint(2, static_cast<uint64_t>(static_cast<int64_t>(*p)));
        w.f_varint(14, P_INT32);
    } else if (auto p = std::get_if<float>(&v)) {
        if (*p != 0.f) w.f_float(3, *p);
        w.f_varint(14, P_FLOAT);
    } else if (auto p = std::get_if<bool>(&v)) {
        if (*p) w.f_varint(4, 1);
        w.f_varint(14, P_BOOLEN);
    } else if (auto p = std::get_if<PTuple<int>>(&v)) {
        Writer c, body;
        for (int x : *p) body.varint(static_cast<uint64_t>(static_cast<int64_t>(x)));
        if (!p->empty()) c.f_bytes(2, body.buf);
        c.f_varint(6, P_INT32);
        if (!p->empty()) c.f_varint(7, p->size());
        w.f_bytes(8, c.buf);
        w.f_varint(14, P_CACHE_LIST);
    } else if (auto p = std::get_if<PTuple<float>>(&v)) {
        Writer c;
        write_cache_floats(c, p->data(), p->size());
        w.f_bytes(8, c.buf);
        w.f_varint(14, P_CACHE_LIST);
    } else if (auto p = std::get_if<PTuple<bool>>(&v)) {
        Writer c; std::string body;
        for (bool x : *p) body.push_back(x ? 1 : 0);
        if (!p->empty()) c.f_bytes(4, body);
        c.f_varint(6, P_BOOLEN);
        if (!p->empty()) c.f_varint(7, p->size());
        w.f_bytes(8, c.buf);
        w.f_varint(14, P_CACHE_LIST);
    } else if (auto p = std::get_if<PTuple<std::string>>(&v)) {
        Writer c;
        for (auto& x : *p) c.f_bytes(1, x);
        if (!p->empty()) c.f_varint(7, p->size());
        w.f_bytes(8, c.buf);
        w.f_varint(14, P_CACHE_LIST);
    } else if (auto p = std::get_if<PBlockPtr>(&v)) {
        Writer t;
        if (share_from && !share_from->empty()) {
            // graph.cpp:700-718 (save): a shared weight is written as a reference to its owner node
            t.f_varint(2, 1);
            t.f_bytes(3, *share_from);
        } else {
            const PBlock& b = **p;
            std::vector<int> dims = {b.h.num(), b.h.channel(), b.h.height(), b.h.width()};
            t.f_bytes(8, enc_shape(dims));
            t.f_bytes(9, enc_shape(dims));
            Writer c;
            const size_t n = static_cast<size_t>(b.count());
            if (b.is_int8()) {
                if (n) c.f_bytes(8, b.h.data(), n);
                c.f_varint(6, P_INT8);
                if (n) c.f_varint(7, n);
            } else {
                write_cache_floats(c, b.data(), n);
            }
            t.f_bytes(10, c.buf);
            if (!b.h.get_scale().empty()) {
                Writer sc;
                write_cache_floats(sc, b.h.get_scale().data(), b.h.get_scale().size());
                t.f_bytes(11, sc.buf);
            }
        }
        w.f_bytes(10, t.buf);
        w.f_varint(14, P_TENSOR);
    }
    return w.buf;
}

}  // namespace

// ------------------------------------------------------------------ GraphIO
class GraphIO {
public:
    static Status parse(GraphCore& g, const void* data, size_t len);
    static std::string serialize(GraphCore& g);
};

Status GraphIO::parse(GraphCore& g, const void* data, size_t len) {
    g._nodes.clear(); g._order.clear(); g._ins.clear(); g._outs.clear(); g._edges.clear();
    std::map<std::string, std::vector<std::pair<std::string, std::vector<float>>>> edges_in, edges_out;
    Reader r(data, len);
    int field, wt; uint64_t v; Reader sub(nullptr, 0);
    bool is_optimized = false;
    while (r.next(field, wt, v, sub)) {
        if (field == 1) {
            g._name = sub.str();
        } else if (field == 2) {  // NodeProto
            NodePtr n = std::make_shared<Node>();
            int f2, w2; uint64_t v2; Reader s2(nullptr, 0);
            while (sub.next(f2, w2, v2, s2)) {
                switch (f2) {
                    case 1: n->name = s2.str(); break;
                    case 2: n->ins.push_back(s2.str()); break;
                    case 3: n->outs.push_back(s2.str()); break;
                    case 10: {
                        std::string key, from, err; AttrValue val; bool got = false;
                        int f3, w3; uint64_t v3; Reader s3(nullptr, 0);
                        while (s2.next(f3, w3, v3, s3)) {
                            if (f3 == 1) key = s3.str();
                            else if (f3 == 2) got = read_value(s3, val, &from, &err);
                        }
                        if (!got) return Status::ANAKINFAIL("bad attr " + key + " in node " + n->name + (err.empty() ? "" : ": " + err));
                        n->attrs[key] = val;
                        if (!from.empty()) n->share_pairs[key] = from;
                    } break;
                    case 11: n->lane = static_cast<int>(v2); break;
                    case 12: n->need_wait = v2 != 0; break;
                    case 15: {
                        int f3, w3; uint64_t v3; Reader s3(nullptr, 0);
                        while (s2.next(f3, w3, v3, s3)) if (f3 == 1) n->op = s3.str();
                    } break;
                    case 16:
                        n->bit_type = (v2 == P_INT8) ? saber::AK_INT8 : (v2 == P_FLOAT ? saber::AK_FLOAT : saber::AK_INVALID);
                        break;
                    default: break;
                }
            }
            if (!sub.ok) return Status::ANAKINFAIL("malformed NodeProto");
            g.add_node(n);
        } else if (field == 3 || field == 4) {  // map<string, List>
            std::string key;
            std::vector<std::pair<std::string, std::vector<float>>> lst;
            int f2, w2; uint64_t v2; Reader s2(nullptr, 0);
            while (sub.next(f2, w2, v2, s2)) {
                if (f2 == 1) key = s2.str();
                else if (f2 == 2) {
                    int f3, w3; uint64_t v3; Reader s3(nullptr, 0);
                    while (s2.next(f3, w3, v3, s3)) {
                        if (f3 == 1) lst.push_back({s3.str(), {}});
                        else if (f3 == 2) {  // TargetProto
                            std::string node; std::vector<float> scale;
                            int f4, w4; uint64_t v4; Reader s4(nullptr, 0);
                            while (s3.next(f4, w4, v4, s4)) {
                                if (f4 == 1) node = s4.str();
                                else if (f4 == 2) {
                                    if (w4 == 2) {
                                        size_t n = static_cast<size_t>(s4.end - s4.p) / 4, o = scale.size();
                                        scale.resize(o + n);
                                        memcpy(scale.data() + o, s4.p, n * 4);
                                    } else { uint32_t u = static_cast<uint32_t>(v4); float f; memcpy(&f, &u, 4); scale.push_back(f); }
                                }
                            }
                            lst.push_back({node, scale});
                        }
                    }
                }
            }
            (field == 3 ? edges_in : edges_out)[key] = lst;
        } else if (field == 6) {
            g._ins.push_back(sub.str());
        } else if (field == 7) {
            g._outs.push_back(sub.str());
        } else if (field == 11) {
            int f2, w2; uint64_t v2; Reader s2(nullptr, 0);
            while (sub.next(f2, w2, v2, s2)) if (f2 == 10) is_optimized = v2 != 0;
        }
    }
    if (!r.ok) return Status::ANAKINFAIL("malformed GraphProto");
    // shared weights: the attribute points at the owner node's block of the same key (model_io.cpp:147-151;
    // resolved after all nodes are read, so the owner may also follow its users in the file)
    for (auto& kv : g._nodes) {
        for (auto& sp : kv.second->share_pairs) {
            NodePtr owner = g[sp.second];
            if (!owner || !owner->has_attr<PBlockPtr>(sp.first) || !owner->get_attr<PBlockPtr>(sp.first) ||
                owner->share_pairs.count(sp.first))
                return Status::ANAKINFAIL("node " + kv.first + " shares '" + sp.first + "' from " + sp.second +
                                          ", which does not own such a tensor");
            kv.second->attrs[sp.first] = owner->get_attr<PBlockPtr>(sp.first);
        }
    }
    // arcs: the edges_in / edges_out maps are authoritative (parser.cpp:160-227)
    for (auto& kv : edges_in) {
        NodePtr n = g[kv.first];
        if (!n) return Status::ANAKINFAIL("edges_in names unknown node " + kv.first);
        n->ins.clear();
        for (auto& t : kv.second) {
            n->ins.push_back(t.first);
            Edge e; e.bottom = t.first; e.top = kv.first; e.scale = t.second;
            g._edges[e.name()] = e;
        }
    }
    for (auto& kv : edges_out) {
        NodePtr n = g[kv.first];
        if (!n) return Status::ANAKINFAIL("edges_out names unknown node " + kv.first);
        n->outs.clear();
        for (auto& t : kv.second) {
            n->outs.push_back(t.first);
            Edge e; e.bottom = kv.first; e.top = t.first; e.scale = t.second;
            auto it = g._edges.find(e.name());
            if (it == g._edges.end()) g._edges[e.name()] = e;
            else if (it->second.scale.empty()) it->second.scale = e.scale;
        }
    }
    for (auto& kv : g._nodes)
        for (auto& b : kv.second->ins)
            if (!g.has_node(b)) return Status::ANAKINFAIL("node " + kv.first + " reads unknown node " + b);
    if (g._ins.empty())
        for (auto& nm : g._order) if (g[nm]->op == "Input") g._ins.push_back(nm);
    if (g._outs.empty())
        for (auto& nm : g._order) if (g[nm]->op == "Output") g._outs.push_back(nm);
    g._optimized = false;  // Optimize force-overrides IS_OPTIMIZED (graph.cpp:359-360)
    (void)is_optimized;
    return Status::OK();
}

std::string GraphIO::serialize(GraphCore& g) {
    Writer w;
    w.f_bytes(1, g._name);
    for (auto& nm : g._order) {
        const Node& n = *g._nodes[nm];
        Writer nw;
        nw.f_bytes(1, n.name);
        for (auto& s : n.ins) nw.f_bytes(2, s);
        for (auto& s : n.outs) nw.f_bytes(3, s);
        for (auto& kv : n.attrs) {
            Writer e;
            e.f_bytes(1, kv.first);
            auto sp = n.share_pairs.find(kv.first);
            e.f_bytes(2, enc_value(kv.second, sp == n.share_pairs.end() ? nullptr : &sp->second));
            nw.f_bytes(10, e.buf);
        }
        if (n.lane) nw.f_varint(11, static_cast<uint64_t>(n.lane));
        if (n.need_wait) nw.f_varint(12, 1);
        Writer op;
        op.f_bytes(1, n.op);
        if (!n.ins.empty()) op.f_varint(3, n.ins.size());     // proto3: zero scalars are not emitted
        if (!n.outs.empty()) op.f_varint(4, n.outs.size());
        nw.f_bytes(15, op.buf);
        if (n.bit_type == saber::AK_INT8) nw.f_varint(16, P_INT8);
        else if (n.bit_type == saber::AK_FLOAT) nw.f_varint(16, P_FLOAT);
        w.f_bytes(2, nw.buf);
    }
    auto enc_list = [&](const std::string& self, const std::vector<std::string>& others, bool in) {
        Writer l;
        for (auto& o : others) {
            std::vector<float> sc = in ? g.edge_scale(o, self) : g.edge_scale(self, o);
            if (sc.empty()) {
                l.f_bytes(1, o);
            } else {
                Writer t;
                t.f_bytes(1, o);
                t.f_bytes(2, sc.data(), sc.size() * 4);
                t.f_varint(3, 8);  // LP_NCHW
                l.f_bytes(2, t.buf);
            }
        }
        return l.buf;
    };
    for (int pass = 0; pass < 2; ++pass) {
        for (auto& nm : g._order) {
            const Node& n = *g._nodes[nm];
            const auto& others = pass == 0 ? n.ins : n.outs;
            if (others.empty()) continue;
            Writer e;
            e.f_bytes(1, nm);
            e.f_bytes(2, enc_list(nm, others, pass == 0));
            w.f_bytes(pass == 0 ? 3 : 4, e.buf);
        }
    }
    for (auto& s : g._ins) w.f_bytes(6, s);
    for (auto& s : g._outs) w.f_bytes(7, s);
    Writer ver;
    ver.f_varint(1, 2);
    ver.f_varint(4, 200);
    w.f_bytes(10, ver.buf);
    Writer info;
    if (g._optimized) info.f_varint(10, 1);
    w.f_bytes(11, info.buf);
    return w.buf;
}

// ------------------------------------------------------------------ GraphCore
void GraphCore::add_node(const NodePtr& n) {
    if (!_nodes.count(n->name)) _order.push_back(n->name);
    _nodes[n->name] = n;
}

void GraphCore::remove_node(const std::string& n) {
    _nodes.erase(n);
    _order.erase(std::remove(_order.begin(), _order.end(), n), _order.end());
}

Status GraphCore::load(const std::string& model_path) {
    std::lock_guard<std::mutex> lk(_mut);
    std::ifstream f(model_path, std::ios::binary | std::ios::ate);
    if (!f) return Status::ANAKINFAIL("cannot open model file " + model_path);
    std::streamsize n = f.tellg();
    f.seekg(0);
    std::string buf(static_cast<size_t>(n), '\0');
    if (n && !f.read(&buf[0], n)) return Status::ANAKINFAIL("short read on " + model_path);
    return GraphIO::parse(*this, buf.data(), buf.size());
}

Status GraphCore::load(const char* buffer, size_t len) {
    std::lock_guard<std::mutex> lk(_mut);
    return GraphIO::parse(*this, buffer, len);
}

Status GraphCore::save(const std::string& model_path) {
    std::lock_guard<std::mutex> lk(_mut);
    std::string s = GraphIO::serialize(*this);
    std::ofstream f(model_path, std::ios::binary);
    if (!f) return Status::ANAKINFAIL("cannot write " + model_path);
    f.write(s.data(), static_cast<std::streamsize>(s.size()));
    return f ? Status::OK() : Status::ANAKINFAIL("short write on " + model_path);
}

void GraphCore::Reshape(const std::string& in_name, std::vector<int> shape) {
    NodePtr n = (*this)[in_name];
    if (!n || n->op != "Input") { fprintf(stderr, "[FATAL] Reshape: no input node %s\n", in_name.c_str()); abort(); }
    n->set_attr("input_shape", PTuple<int>(shape));
}

void GraphCore::ResetBatchSize(const std::string& in_name, int batch_size) {
    NodePtr n = (*this)[in_name];
    if (!n || n->op != "Input") { fprintf(stderr, "[FATAL] ResetBatchSize: no input node %s\n", in_name.c_str()); abort(); }
    PTuple<int> s = n->get_attr<PTuple<int>>("input_shape");
    if (s.empty()) s = {1, 1, 1, 1};
    s[0] = batch_size;
    n->set_attr("input_shape", s);
}

namespace {
int input_channels(const Node& n) {
    const PTuple<int> s = n.get_attr_or<PTuple<int>>("input_shape", {});
    return s.size() >= 2 ? s[1] : 1;
}
}  // namespace

int node_image_format(const Node& n, b200_image_desc_t* fmt) {
    if (!n.has("image_src_channel") && !n.has("image_mean") && !n.has("image_scale")) return 0;
    const PTuple<int> src = n.get_attr_or<PTuple<int>>("image_src_channel", {});
    const PTuple<float> mean = n.get_attr_or<PTuple<float>>("image_mean", {});
    const PTuple<float> scale = n.get_attr_or<PTuple<float>>("image_scale", {});
    const int c = input_channels(n);
    if (c < 1 || c > 4 || static_cast<int>(src.size()) != c || mean.size() != src.size() || scale.size() != src.size())
        return -1;
    b200_image_desc_t d;
    memset(&d, 0, sizeof(d));
    for (int i = 0; i < c; ++i) { d.src_channel[i] = src[i]; d.mean[i] = mean[i]; d.scale[i] = scale[i]; }
    if (!b200_image_desc_valid(&d, c)) return -1;
    if (fmt) *fmt = d;
    return 1;
}

Status GraphCore::set_input_image(const std::string& in_name, const b200_image_desc_t& fmt) {
    NodePtr n = (*this)[in_name];
    if (!n) return Status::ANAKINFAIL("set_input_image: no node " + in_name);
    if (n->op != "Input") return Status::ANAKINFAIL("set_input_image: node " + in_name + " is a " + n->op + ", not an Input");
    const int c = input_channels(*n);
    if (!b200_image_desc_valid(&fmt, c))
        return Status::ANAKINFAIL("set_input_image(" + in_name + "): invalid format for " + std::to_string(c) +
                                  " channels (1..4 channels, src_channel a permutation of 0..c-1, finite mean and scale)");
    n->set_attr("image_src_channel", PTuple<int>(fmt.src_channel, fmt.src_channel + c));
    n->set_attr("image_mean", PTuple<float>(fmt.mean, fmt.mean + c));
    n->set_attr("image_scale", PTuple<float>(fmt.scale, fmt.scale + c));
    return Status::OK();
}

bool GraphCore::input_image(const std::string& in_name, b200_image_desc_t* fmt) const {
    NodePtr n = (*this)[in_name];
    return n && n->op == "Input" && node_image_format(*n, fmt) == 1;
}

int node_image_resize(const Node& n, ImageResize* r) {
    if (!n.has("image_max_h") && !n.has("image_max_w") && !n.has("image_resize_short")) return 0;
    ImageResize v;
    v.max_h = n.get_attr_or<int>("image_max_h", 0);
    v.max_w = n.get_attr_or<int>("image_max_w", 0);
    v.resize_short = n.get_attr_or<int>("image_resize_short", -1);
    if (v.max_h < 1 || v.max_h > ImageResize::kMaxSide || v.max_w < 1 || v.max_w > ImageResize::kMaxSide ||
        v.resize_short < 0)
        return -1;
    if (r) *r = v;
    return 1;
}

Status GraphCore::set_input_image_resize(const std::string& in_name, int max_h, int max_w, int resize_short) {
    NodePtr n = (*this)[in_name];
    if (!n) return Status::ANAKINFAIL("set_input_image_resize: no node " + in_name);
    if (n->op != "Input")
        return Status::ANAKINFAIL("set_input_image_resize: node " + in_name + " is a " + n->op + ", not an Input");
    if (node_image_format(*n, nullptr) != 1)
        return Status::ANAKINFAIL("set_input_image_resize(" + in_name + "): not an image input (call set_input_image first)");
    if (max_h < 1 || max_h > ImageResize::kMaxSide || max_w < 1 || max_w > ImageResize::kMaxSide)
        return Status::ANAKINFAIL("set_input_image_resize(" + in_name + "): max_h and max_w must be in 1.." +
                                  std::to_string(ImageResize::kMaxSide) + ", got " + std::to_string(max_h) + " x " +
                                  std::to_string(max_w));
    if (resize_short < 0)
        return Status::ANAKINFAIL("set_input_image_resize(" + in_name + "): resize_short must be >= 0, got " +
                                  std::to_string(resize_short));
    n->set_attr("image_max_h", max_h);
    n->set_attr("image_max_w", max_w);
    n->set_attr("image_resize_short", resize_short);
    return Status::OK();
}

bool GraphCore::input_image_resize(const std::string& in_name, ImageResize* r) const {
    NodePtr n = (*this)[in_name];
    return n && n->op == "Input" && node_image_resize(*n, r) == 1;
}

std::vector<float> GraphCore::edge_scale(const std::string& bottom, const std::string& top) const {
    auto it = _edges.find(bottom + "_" + top);
    if (it != _edges.end()) return it->second.scale;
    return {};
}

std::vector<float> GraphCore::node_out_scale(const std::string& node) const {
    auto it = _nodes.find(node);
    if (it == _nodes.end()) return {};
    for (auto& t : it->second->outs) {
        std::vector<float> s = edge_scale(node, t);
        if (!s.empty()) return s;
    }
    return {};
}

Status GraphCore::AddOp(const std::string& name, const std::string& type, const std::vector<std::string>& ins,
                        const std::vector<std::string>& outs) {
    if (_nodes.count(name)) return Status::ANAKINFAIL("duplicate op " + name);
    NodePtr n = std::make_shared<Node>();
    n->name = name; n->op = type; n->ins = ins; n->outs = outs;
    add_node(n);
    return Status::OK();
}

Status GraphCore::Freeze() {
    // derive outs from ins so a hand-built graph only has to name its producers
    for (auto& kv : _nodes) kv.second->outs.clear();
    for (auto& nm : _order)
        for (auto& b : _nodes[nm]->ins) {
            if (!_nodes.count(b)) return Status::ANAKINFAIL("op " + nm + " reads unknown op " + b);
            _nodes[b]->outs.push_back(nm);
        }
    _ins.clear(); _outs.clear();
    for (auto& nm : _order) {
        if (_nodes[nm]->op == "Input") _ins.push_back(nm);
        if (_nodes[nm]->op == "Output") _outs.push_back(nm);
    }
    rebuild_edges_from_nodes();
    return Status::OK();
}

void GraphCore::rebuild_edges_from_nodes() {
    std::map<std::string, Edge> fresh;
    for (auto& nm : _order)
        for (auto& t : _nodes[nm]->outs) {
            Edge e; e.bottom = nm; e.top = t;
            auto it = _edges.find(e.name());
            if (it != _edges.end()) e.scale = it->second.scale;
            fresh[e.name()] = e;
        }
    _edges.swap(fresh);
}

Status GraphCore::topo_sort() {
    std::map<std::string, int> indeg, rank;
    for (size_t i = 0; i < _order.size(); ++i) rank[_order[i]] = static_cast<int>(i);
    for (auto& kv : _nodes) indeg[kv.first] = static_cast<int>(kv.second->ins.size());
    auto cmp = [&](const std::string& a, const std::string& b) { return rank[a] < rank[b]; };
    std::set<std::string, decltype(cmp)> ready(cmp);
    for (auto& kv : indeg) if (kv.second == 0) ready.insert(kv.first);
    std::vector<std::string> out;
    while (!ready.empty()) {
        std::string n = *ready.begin();
        ready.erase(ready.begin());
        out.push_back(n);
        for (auto& t : _nodes[n]->outs)
            if (--indeg[t] == 0) ready.insert(t);
    }
    if (out.size() != _nodes.size()) return Status::ANAKINFAIL("graph has a cycle or dangling arcs");
    _order.swap(out);
    return Status::OK();
}

// ---- in-order fusion patterns (fusion_op_register.cpp:45-175), longest first
namespace {
struct Pattern {
    const char* fused;
    std::vector<std::pair<const char*, const char*>> chain;  // (pattern node name, op)
};
const std::vector<Pattern>& patterns() {
    static const std::vector<Pattern> p = {
        {"ConvBatchnormScaleReluPool", {{"conv_0", "Convolution"}, {"batchnorm_0", "BatchNorm"}, {"scale_0", "Scale"}, {"relu_0", "ReLU"}, {"pooling_0", "Pooling"}}},
        {"ConvBatchnormScaleRelu", {{"conv_0", "Convolution"}, {"batchnorm_0", "BatchNorm"}, {"scale_0", "Scale"}, {"relu_0", "ReLU"}}},
        {"ConvReluPool", {{"conv_0", "Convolution"}, {"relu_0", "ReLU"}, {"pooling_0", "Pooling"}}},
        {"ConvBatchnormScale", {{"conv_0", "Convolution"}, {"batchnorm_0", "BatchNorm"}, {"scale_0", "Scale"}}},
        {"ConvScaleRelu", {{"conv_0", "Convolution"}, {"scale_0", "Scale"}, {"relu_0", "ReLU"}}},
        {"ConvBatchnorm", {{"conv_0", "Convolution"}, {"batchnorm_0", "BatchNorm"}}},
        {"ConvScale", {{"conv_0", "Convolution"}, {"scale_0", "Scale"}}},
        {"ConvRelu", {{"conv_0", "Convolution"}, {"relu_0", "ReLU"}}},
        {"EltwiseRelu", {{"eltwise_0", "Eltwise"}, {"relu_0", "ReLU"}}},
    };
    return p;
}
}  // namespace

void GraphCore::fuse_in_order_patterns() {
    for (const Pattern& pat : patterns()) {
        const bool has_pool = std::string(pat.fused).find("Pool") != std::string::npos;
        std::vector<std::string> order_copy = _order;
        for (auto& head_name : order_copy) {
            if (!_nodes.count(head_name)) continue;
            NodePtr head = _nodes[head_name];
            if (head->op != pat.chain[0].second) continue;
            // Conv*Pool fusions: the reference skips them for NV-INT8 (graph.cpp:378-386) -- its INT8 conv has no fused
            // pooling kernel. Here an INT8 conv absorbs a following MAX pooling (the stem kernel runs both in one launch;
            // int8 pooling passes its input scale through, saber_pooling.cpp:583-584, so the fused node's output simply
            // carries the conv's output scale). B200_ANAKIN_INT8_CONV_POOL=0 restores the reference behaviour.
            const bool int8_head = head->bit_type == saber::AK_INT8;
            static const bool int8_pool_fusion = [] { const char* e = getenv("B200_ANAKIN_INT8_CONV_POOL"); return !(e && e[0] == '0'); }();
            if (has_pool && int8_head && !int8_pool_fusion) continue;
            std::vector<NodePtr> chain = {head};
            bool ok = true;
            for (size_t i = 1; i < pat.chain.size(); ++i) {
                NodePtr cur = chain.back();
                if (cur->outs.size() != 1) { ok = false; break; }
                NodePtr nxt = _nodes[cur->outs[0]];
                if (!nxt || nxt->op != pat.chain[i].second || nxt->ins.size() != 1) { ok = false; break; }
                chain.push_back(nxt);
            }
            if (!ok) continue;
            if (has_pool && int8_head) {
                const NodePtr& pool = chain.back();
                if (pool->get_attr_or<std::string>("method", "") != "MAX" || pool->get_attr_or<bool>("global_pooling", false))
                    continue;
            }
            // merge attrs of the followers into the head with prefix "<patternNode>_" (graph.cpp:588-762)
            for (size_t i = 1; i < chain.size(); ++i) {
                const std::string prefix = std::string(pat.chain[i].first) + "_";
                for (auto& kv : chain[i]->attrs) head->attrs[prefix + kv.first] = kv.second;
            }
            NodePtr last = chain.back();
            // the fused node's output edge inherits the last node's edges (and scales)
            for (auto& t : last->outs) {
                Edge e; e.bottom = head->name; e.top = t;
                e.scale = edge_scale(last->name, t);
                if (has_pool && int8_head) {   // the tensor the fused node writes is requantised with the conv's output scale
                    std::vector<float> s_in = edge_scale(chain[chain.size() - 2]->name, last->name);
                    if (!s_in.empty()) e.scale = s_in;
                }
                _edges[e.name()] = e;
                for (auto& b : _nodes[t]->ins) if (b == last->name) b = head->name;
            }
            head->outs = last->outs;
            head->op = pat.fused;
            for (size_t i = 1; i < chain.size(); ++i) remove_node(chain[i]->name);
        }
    }
}

// ConvEltwise (conv_elewise_fusion_scheduler.cpp:31-136): conv-without-activation whose only
// consumer is an Eltwise Add (coeff 1,1) [+ReLU] absorbs it; the other eltwise input becomes the
// conv's second input (the residual), which therefore executes first. The reference gates this
// pass to FP32 (graph.cpp:428); it is enabled for INT8 here as BASELINE north_star asks.
void GraphCore::fuse_conv_eltwise() {
    static const std::set<std::string> conv_ops = {"Convolution", "ConvBatchnormScale", "ConvBatchnorm", "ConvScale"};
    std::map<std::string, int> rank;
    for (size_t i = 0; i < _order.size(); ++i) rank[_order[i]] = static_cast<int>(i);
    std::vector<std::string> order_copy = _order;
    for (auto& en : order_copy) {
        if (!_nodes.count(en)) continue;
        NodePtr elt = _nodes[en];
        if (elt->op != "Eltwise" && elt->op != "EltwiseRelu") continue;
        if (elt->ins.size() != 2) continue;
        if (elt->get_attr_or<std::string>("type", "") != "Add") continue;
        PTuple<float> coeff = elt->get_attr_or<PTuple<float>>("coeff", {});
        bool unit = true;
        for (float c : coeff) if (c != 1.f) unit = false;
        if (!unit) continue;
        NodePtr best;
        for (auto& b : elt->ins) {
            NodePtr p = _nodes[b];
            if (!conv_ops.count(p->op) || p->outs.size() != 1 || p->ins.size() != 1) continue;
            if (p->get_attr_or<int>("group", 1) != 1) continue;
            if (!best || rank[p->name] > rank[best->name]) best = p;
        }
        if (!best) continue;
        std::string other;
        for (auto& b : elt->ins) if (b != best->name) other = b;
        if (other.empty()) continue;
        for (auto& kv : elt->attrs) best->attrs["merge_" + kv.first] = kv.second;
        best->attrs["conv_eltwise_base_op"] = best->op;  // which conv flavour was absorbed
        best->op = "ConvEltwise";
        best->ins.push_back(other);
        // the residual producer now feeds the conv instead of the eltwise
        for (auto& t : _nodes[other]->outs) if (t == elt->name) t = best->name;
        {
            Edge e; e.bottom = other; e.top = best->name; e.scale = edge_scale(other, elt->name);
            _edges[e.name()] = e;
        }
        for (auto& t : elt->outs) {
            Edge e; e.bottom = best->name; e.top = t; e.scale = edge_scale(elt->name, t);
            _edges[e.name()] = e;
            for (auto& b : _nodes[t]->ins) if (b == elt->name) b = best->name;
        }
        best->outs = elt->outs;
        remove_node(elt->name);
    }
}

Status GraphCore::Optimize(bool with_fusion) {
    std::lock_guard<std::mutex> lk(_mut);
    Status st = topo_sort();
    if (!st) return st;
    if (with_fusion) {
        fuse_in_order_patterns();
        st = topo_sort();
        if (!st) return st;
        fuse_conv_eltwise();
    }
    st = topo_sort();
    if (!st) return st;
    rebuild_edges_from_nodes();
    _optimized = true;
    return Status::OK();
}

}  // namespace graph
}  // namespace anakin
