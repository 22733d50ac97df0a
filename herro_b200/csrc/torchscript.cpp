// Reader for TorchScript archives (`torch.jit.save`): what `-m model.pt` names in the reference CLI (src/main.rs, loaded by
// tch::CModule::load_on_device at src/inference.rs:185).  The library does not execute TorchScript; it takes the parameters of
// a module with the architecture it implements (herro_b200/weights.py, oracle/forward_ref.py naming) out of the archive:
//   * the archive is a ZIP whose entries are stored uncompressed (PyTorch's writer never compresses): central directory,
//     ZIP64 records when present;
//   * `<name>/data.pkl` is a protocol-2 pickle of the module object tree: objects are NEWOBJ + BUILD(dict of attributes),
//     tensors are REDUCE(torch._utils._rebuild_tensor_v2, (persistent-id storage, offset, size, stride, requires_grad, hooks)),
//     storages are persistent ids ('storage', torch.<T>Storage, key, device, numel) whose bytes live in `<name>/data/<key>`;
//   * attribute paths ("layers.0.qkv.weight") are the state_dict names.
// Only what such archives contain is interpreted; anything else is an error (HB_ERR_MODEL), never a guess.
#include "torchscript.h"

#include <cmath>
#include <cstring>
#include <memory>
#include <unordered_map>

namespace hb {
namespace {

uint16_t rd16(const uint8_t* p) { return (uint16_t)(p[0] | (p[1] << 8)); }
uint32_t rd32(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }
uint64_t rd64(const uint8_t* p) { return (uint64_t)rd32(p) | ((uint64_t)rd32(p + 4) << 32); }

struct ZipEntry { uint64_t off = 0, size = 0; bool compressed = false; };

// name -> (offset of the data, size) for every stored entry
bool zip_index(const uint8_t* b, size_t n, std::unordered_map<std::string, ZipEntry>& out, std::string& err) {
    if (n < 22) { err = "archive too small"; return false; }
    size_t eocd = (size_t)-1;
    const size_t lo = n > (size_t)(22 + 65535) ? n - (22 + 65535) : 0;
    for (size_t i = n - 22 + 1; i-- > lo;)
        if (rd32(b + i) == 0x06054b50u) { eocd = i; break; }
    if (eocd == (size_t)-1) { err = "no ZIP end-of-central-directory record"; return false; }
    uint64_t n_ent = rd16(b + eocd + 10), cd_size = rd32(b + eocd + 12), cd_off = rd32(b + eocd + 16);
    if (n_ent == 0xffff || cd_size == 0xffffffffu || cd_off == 0xffffffffu) {  // ZIP64
        if (eocd < 20 || rd32(b + eocd - 20) != 0x07064b50u) { err = "ZIP64 locator missing"; return false; }
        const uint64_t z = rd64(b + eocd - 20 + 8);
        if (z > n || n - z < 56 || rd32(b + z) != 0x06064b50u) { err = "bad ZIP64 end-of-central-directory record"; return false; }
        n_ent = rd64(b + z + 32); cd_size = rd64(b + z + 40); cd_off = rd64(b + z + 48);
    }
    if (cd_off > n || cd_size > n - cd_off || n_ent > (1u << 20)) { err = "central directory out of bounds"; return false; }
    size_t p = (size_t)cd_off;
    const size_t end = (size_t)(cd_off + cd_size);
    for (uint64_t e = 0; e < n_ent; e++) {
        if (end - p < 46 || rd32(b + p) != 0x02014b50u) { err = "bad central directory entry"; return false; }
        const uint16_t method = rd16(b + p + 10), nl = rd16(b + p + 28), xl = rd16(b + p + 30), cl = rd16(b + p + 32);
        uint64_t csize = rd32(b + p + 20), usize = rd32(b + p + 24), lho = rd32(b + p + 42);
        if ((size_t)46 + nl + xl + cl > end - p) { err = "bad central directory entry"; return false; }
        const std::string name((const char*)b + p + 46, nl);
        // ZIP64 extended information: the fields that are 0xffffffff in the fixed part, in this order
        for (size_t x = p + 46 + nl, xe = x + xl; x + 4 <= xe;) {
            const uint16_t id = rd16(b + x), len = rd16(b + x + 2);
            if (x + 4 + len > xe) break;
            if (id == 1) {
                size_t q = x + 4;
                if (usize == 0xffffffffu && q + 8 <= x + 4 + len) { usize = rd64(b + q); q += 8; }
                if (csize == 0xffffffffu && q + 8 <= x + 4 + len) { csize = rd64(b + q); q += 8; }
                if (lho == 0xffffffffu && q + 8 <= x + 4 + len) { lho = rd64(b + q); q += 8; }
            }
            x += 4 + (size_t)len;
        }
        p += (size_t)46 + nl + xl + cl;
        if (!name.empty() && name.back() == '/') continue;
        if (method != 0 || csize != usize) { out[name] = ZipEntry{0, 0, true}; continue; }  // PyTorch deflates only code/*.py: never needed here
        if (lho > n || n - lho < 30 || rd32(b + lho) != 0x04034b50u) { err = "bad local header of '" + name + "'"; return false; }
        const uint64_t data = lho + 30 + rd16(b + lho + 26) + rd16(b + lho + 28);
        if (data > n || usize > n - data) { err = "entry '" + name + "' out of bounds"; return false; }
        out[name] = ZipEntry{data, usize, false};
    }
    return true;
}

// ---- pickle values ----------------------------------------------------------------------------------------------------
struct PV;
using PVP = std::shared_ptr<PV>;
struct PV {
    enum Kind { NONE, BOOL, INT, FLOAT, STR, TUPLE, LIST, DICT, GLOBAL, OBJ, TENSOR, STORAGE, MARK } k = NONE;
    int64_t i = 0;                 // BOOL / INT; STORAGE: numel; TENSOR: storage offset (elements)
    double f = 0;                  // FLOAT
    std::string s;                 // STR / GLOBAL ("module name") / STORAGE: key
    std::string dtype;             // STORAGE: torch storage class
    std::vector<PVP> items;        // TUPLE / LIST; DICT: key, value, key, value, ...
    PVP cls, state;                // OBJ
    PVP storage;                   // TENSOR
    std::vector<int64_t> shape, stride;
};
PVP mk(PV::Kind k) { auto p = std::make_shared<PV>(); p->k = k; return p; }

bool ints_of(const PVP& t, std::vector<int64_t>& out) {
    if (!t || t->k != PV::TUPLE) return false;
    for (auto& e : t->items) {
        if (!e || e->k != PV::INT) return false;
        out.push_back(e->i);
    }
    return true;
}

bool unpickle(const uint8_t* b, size_t n, PVP& root, std::string& err) {
    std::vector<PVP> st;
    std::unordered_map<uint32_t, PVP> memo;
    size_t p = 0;
    auto need = [&](size_t k) { return n - p >= k; };
    auto pop = [&](PVP& v) -> bool { if (st.empty() || st.back()->k == PV::MARK) return false; v = st.back(); st.pop_back(); return true; };
    auto pop_mark = [&](std::vector<PVP>& items) -> bool {
        size_t m = st.size();
        while (m > 0 && st[m - 1]->k != PV::MARK) m--;
        if (m == 0) return false;
        items.assign(st.begin() + (long)m, st.end());
        st.resize(m - 1);
        return true;
    };
    auto line = [&](std::string& out) -> bool {
        const size_t s0 = p;
        while (p < n && b[p] != '\n') p++;
        if (p >= n) return false;
        out.assign((const char*)b + s0, p - s0);
        p++;
        return true;
    };
    size_t ops = 0;
    while (p < n) {
        if (++ops > (1u << 22) || st.size() > (1u << 20)) { err = "pickle too large"; return false; }
        const uint8_t op = b[p++];
        switch (op) {
        case 0x80: if (!need(1)) goto trunc; if (b[p] > 5) { err = "pickle protocol too new"; return false; } p++; break;  // PROTO
        case 0x95: if (!need(8)) goto trunc; p += 8; break;                                                           // FRAME
        case '.': { if (!pop(root)) { err = "empty pickle"; return false; } return true; }
        case '(': st.push_back(mk(PV::MARK)); break;
        case 'N': st.push_back(mk(PV::NONE)); break;
        case 0x88: case 0x89: { auto v = mk(PV::BOOL); v->i = (op == 0x88); st.push_back(v); break; }
        case 'K': { if (!need(1)) goto trunc; auto v = mk(PV::INT); v->i = b[p]; p += 1; st.push_back(v); break; }
        case 'M': { if (!need(2)) goto trunc; auto v = mk(PV::INT); v->i = rd16(b + p); p += 2; st.push_back(v); break; }
        case 'J': { if (!need(4)) goto trunc; auto v = mk(PV::INT); v->i = (int32_t)rd32(b + p); p += 4; st.push_back(v); break; }
        case 0x8a: {  // LONG1
            if (!need(1)) goto trunc;
            const uint8_t len = b[p++];
            if (!need(len) || len > 8) { err = "unsupported LONG1"; return false; }
            uint64_t u = 0;
            for (int k = 0; k < len; k++) u |= (uint64_t)b[p + k] << (8 * k);
            if (len && len < 8 && (b[p + len - 1] & 0x80)) u |= ~0ull << (8 * len);
            p += len;
            auto v = mk(PV::INT); v->i = (int64_t)u; st.push_back(v);
            break;
        }
        case 'G': {  // BINFLOAT, big endian
            if (!need(8)) goto trunc;
            uint64_t u = 0;
            for (int k = 0; k < 8; k++) u = (u << 8) | b[p + k];
            p += 8;
            auto v = mk(PV::FLOAT); memcpy(&v->f, &u, 8); st.push_back(v);
            break;
        }
        case 'X': case 0x8c: case 'T': case 'U': case 'B': case 'C': {  // BINUNICODE, SHORT_BINUNICODE, BINSTRING, SHORT_BINSTRING, BINBYTES, SHORT_BINBYTES
            const bool shortf = (op == 0x8c || op == 'U' || op == 'C');
            if (!need(shortf ? 1 : 4)) goto trunc;
            const size_t len = shortf ? b[p] : rd32(b + p);
            p += shortf ? 1 : 4;
            if (!need(len)) goto trunc;
            auto v = mk(PV::STR); v->s.assign((const char*)b + p, len); p += len; st.push_back(v);
            break;
        }
        case 'c': {  // GLOBAL
            std::string m, nm;
            if (!line(m) || !line(nm)) goto trunc;
            auto v = mk(PV::GLOBAL); v->s = m + " " + nm; st.push_back(v);
            break;
        }
        case 0x93: {  // STACK_GLOBAL
            PVP nm, m;
            if (!pop(nm) || !pop(m) || nm->k != PV::STR || m->k != PV::STR) { err = "bad STACK_GLOBAL"; return false; }
            auto v = mk(PV::GLOBAL); v->s = m->s + " " + nm->s; st.push_back(v);
            break;
        }
        case 'q': { if (!need(1) || st.empty()) goto trunc; memo[b[p]] = st.back(); p += 1; break; }
        case 'r': { if (!need(4) || st.empty()) goto trunc; memo[rd32(b + p)] = st.back(); p += 4; break; }
        case 0x94: { if (st.empty()) goto trunc; memo[(uint32_t)memo.size()] = st.back(); break; }  // MEMOIZE
        case 'h': case 'j': {
            if (!need(op == 'h' ? 1 : 4)) goto trunc;
            const uint32_t id = op == 'h' ? b[p] : rd32(b + p);
            p += op == 'h' ? 1 : 4;
            auto it = memo.find(id);
            if (it == memo.end()) { err = "pickle memo miss"; return false; }
            st.push_back(it->second);
            break;
        }
        case ')': st.push_back(mk(PV::TUPLE)); break;
        case ']': st.push_back(mk(PV::LIST)); break;
        case '}': st.push_back(mk(PV::DICT)); break;
        case 't': { auto v = mk(PV::TUPLE); if (!pop_mark(v->items)) goto bad; st.push_back(v); break; }
        case 0x85: case 0x86: case 0x87: {
            const int k = op - 0x84;
            auto v = mk(PV::TUPLE);
            v->items.resize(k);
            for (int q = k - 1; q >= 0; q--) if (!pop(v->items[q])) goto bad;
            st.push_back(v);
            break;
        }
        case 'a': { PVP x; if (!pop(x) || st.empty() || st.back()->k != PV::LIST) goto bad; st.back()->items.push_back(x); break; }
        case 'e': { std::vector<PVP> it; if (!pop_mark(it) || st.empty() || st.back()->k != PV::LIST) goto bad; for (auto& x : it) st.back()->items.push_back(x); break; }
        case 's': { PVP v, k; if (!pop(v) || !pop(k) || st.empty() || st.back()->k != PV::DICT) goto bad; st.back()->items.push_back(k); st.back()->items.push_back(v); break; }
        case 'u': {
            std::vector<PVP> it;
            if (!pop_mark(it) || (it.size() & 1) || st.empty() || st.back()->k != PV::DICT) goto bad;
            for (auto& x : it) st.back()->items.push_back(x);
            break;
        }
        case 0x81: {  // NEWOBJ: cls, args
            PVP args, cls;
            if (!pop(args) || !pop(cls)) goto bad;
            auto v = mk(PV::OBJ); v->cls = cls; st.push_back(v);
            break;
        }
        case 'b': {  // BUILD
            PVP state;
            if (!pop(state) || st.empty()) goto bad;
            if (st.back()->k == PV::OBJ) st.back()->state = state;
            break;
        }
        case 'Q': {  // BINPERSID: ('storage', torch.<T>Storage, key, device, numel[, view])
            PVP pid;
            if (!pop(pid) || pid->k != PV::TUPLE || pid->items.size() < 5 || pid->items[0]->k != PV::STR || pid->items[0]->s != "storage" ||
                pid->items[1]->k != PV::GLOBAL || pid->items[2]->k != PV::STR || pid->items[4]->k != PV::INT) {
                err = "unsupported persistent id in the pickle";
                return false;
            }
            auto v = mk(PV::STORAGE); v->dtype = pid->items[1]->s; v->s = pid->items[2]->s; v->i = pid->items[4]->i; st.push_back(v);
            break;
        }
        case 'R': {  // REDUCE: callable, args
            PVP args, fn;
            if (!pop(args) || !pop(fn) || args->k != PV::TUPLE) goto bad;
            const std::string f = fn->k == PV::GLOBAL ? fn->s : "";
            if (f == "torch._utils _rebuild_tensor_v2" || f == "torch._utils _rebuild_tensor") {
                if (args->items.size() < 4 || args->items[0]->k != PV::STORAGE || args->items[1]->k != PV::INT) { err = "bad _rebuild_tensor arguments"; return false; }
                auto v = mk(PV::TENSOR);
                v->storage = args->items[0]; v->i = args->items[1]->i;
                if (!ints_of(args->items[2], v->shape) || !ints_of(args->items[3], v->stride) || v->shape.size() != v->stride.size()) { err = "bad tensor size/stride"; return false; }
                st.push_back(v);
            } else if (f == "torch._utils _rebuild_parameter" || f == "torch._utils _rebuild_parameter_with_state") {
                if (args->items.empty() || args->items[0]->k != PV::TENSOR) { err = "bad _rebuild_parameter arguments"; return false; }
                st.push_back(args->items[0]);
            } else if (f == "collections OrderedDict") {
                st.push_back(mk(PV::DICT));
            } else {
                auto v = mk(PV::OBJ); v->cls = fn; v->state = args; st.push_back(v);
            }
            break;
        }
        default: err = "unsupported pickle opcode 0x" + std::string(1, "0123456789abcdef"[op >> 4]) + std::string(1, "0123456789abcdef"[op & 15]); return false;
        }
        continue;
    trunc: err = "truncated pickle"; return false;
    bad: err = "malformed pickle (stack)"; return false;
    }
    err = "pickle without STOP";
    return false;
}

float half_to_float(uint16_t h) {
    const uint32_t s = (uint32_t)(h >> 15) << 31, e = (h >> 10) & 31, m = h & 1023;
    uint32_t u;
    if (e == 0) {
        if (m == 0) u = s;
        else { int k = 0; uint32_t mm = m; while (!(mm & 1024)) { mm <<= 1; k++; } u = s | ((uint32_t)(113 - k) << 23) | ((mm & 1023) << 13); }
    } else if (e == 31) u = s | 0x7f800000u | (m << 13);
    else u = s | ((e + 112) << 23) | (m << 13);
    float f; memcpy(&f, &u, 4); return f;
}

}  // namespace

bool ts_is_zip(const uint8_t* buf, size_t n) { return n >= 4 && buf[0] == 'P' && buf[1] == 'K' && buf[2] == 3 && buf[3] == 4; }

bool ts_read_archive(const uint8_t* buf, size_t n, TsModel& out) {
    std::unordered_map<std::string, ZipEntry> zi;
    if (!zip_index(buf, n, zi, out.err)) return false;
    std::string pkl;
    for (auto& kv : zi) {  // "<archive name>/data.pkl": the shortest such path
        const std::string& nm = kv.first;
        if (nm.size() >= 9 && nm.compare(nm.size() - 9, 9, "/data.pkl") == 0 && (pkl.empty() || nm.size() < pkl.size())) pkl = nm;
    }
    if (pkl.empty()) { out.err = "no data.pkl in the archive (not a TorchScript / torch.save archive)"; return false; }
    const std::string root_dir = pkl.substr(0, pkl.size() - 8);  // with the trailing '/'
    if (zi[pkl].compressed) { out.err = "compressed ZIP entry '" + pkl + "' (PyTorch stores data.pkl and the tensor storages uncompressed)"; return false; }
    PVP root;
    if (!unpickle(buf + zi[pkl].off, (size_t)zi[pkl].size, root, out.err)) return false;
    // torch.save of a plain state_dict ({"state_dict": {...}} or the dict itself) is walked the same way
    if (root && root->k == PV::DICT) {
        for (size_t i = 0; i + 1 < root->items.size(); i += 2)
            if (root->items[i]->k == PV::STR && root->items[i]->s == "state_dict") { root = root->items[i + 1]; break; }
    }
    // collect names, then materialise: a second walk that carries the PV nodes
    struct Item { std::string name; PVP t; };
    std::vector<Item> items;
    {
        std::vector<std::pair<PVP, std::string>> stack{{root, ""}};
        size_t guard = 0;
        while (!stack.empty() && ++guard < (1u << 20)) {
            auto cur = stack.back();
            stack.pop_back();
            const PVP& v = cur.first;
            if (!v) continue;
            if (v->k == PV::OBJ) stack.push_back({v->state, cur.second});
            else if (v->k == PV::DICT) {
                for (size_t i = 0; i + 1 < v->items.size(); i += 2)
                    if (v->items[i]->k == PV::STR)
                        stack.push_back({v->items[i + 1], cur.second.empty() ? v->items[i]->s : cur.second + "." + v->items[i]->s});
            } else if (v->k == PV::INT) out.ints[cur.second] = v->i;
            else if (v->k == PV::TENSOR) items.push_back({cur.second, v});
        }
    }
    for (auto& it : items) {
        const PV& t = *it.t;
        const PV& sg = *t.storage;
        auto ze = zi.find(root_dir + "data/" + sg.s);
        if (ze == zi.end()) { out.err = "storage '" + sg.s + "' of tensor " + it.name + " is not in the archive"; return false; }
        if (ze->second.compressed) { out.err = "compressed ZIP entry '" + ze->first + "' (PyTorch stores data.pkl and the tensor storages uncompressed)"; return false; }
        size_t esz;
        int kind;  // 0 f32, 1 f64, 2 f16, 3 bf16
        if (sg.dtype == "torch FloatStorage") { esz = 4; kind = 0; }
        else if (sg.dtype == "torch DoubleStorage") { esz = 8; kind = 1; }
        else if (sg.dtype == "torch HalfStorage") { esz = 2; kind = 2; }
        else if (sg.dtype == "torch BFloat16Storage") { esz = 2; kind = 3; }
        else continue;  // integer buffers (num_batches_tracked, ...) are not parameters of the forward
        const uint64_t n_sto = ze->second.size / esz;
        uint64_t count = 1;
        for (size_t d = 0; d < t.shape.size(); d++) {
            if (t.shape[d] < 0 || t.stride[d] < 0 || (t.shape[d] && count > (1ull << 32) / (uint64_t)t.shape[d])) { out.err = "bad shape of tensor " + it.name; return false; }
            count *= (uint64_t)t.shape[d];
        }
        uint64_t last = (uint64_t)t.i;
        for (size_t d = 0; d < t.shape.size(); d++) if (t.shape[d]) last += (uint64_t)(t.shape[d] - 1) * (uint64_t)t.stride[d];
        if (t.i < 0 || (count && last >= n_sto)) { out.err = "tensor " + it.name + " reaches outside its storage"; return false; }
        TsTensor& dst = out.tensors[it.name];
        dst.shape = t.shape;
        dst.data.resize((size_t)count);
        const uint8_t* base = buf + ze->second.off;
        std::vector<int64_t> idx(t.shape.size(), 0);
        for (uint64_t e = 0; e < count; e++) {
            uint64_t off = (uint64_t)t.i;
            for (size_t d = 0; d < idx.size(); d++) off += (uint64_t)idx[d] * (uint64_t)t.stride[d];
            const uint8_t* q = base + off * esz;
            float v;
            if (kind == 0) memcpy(&v, q, 4);
            else if (kind == 1) { double dd; memcpy(&dd, q, 8); v = (float)dd; }
            else if (kind == 2) v = half_to_float(rd16(q));
            else { const uint32_t u = (uint32_t)rd16(q) << 16; memcpy(&v, &u, 4); }
            dst.data[(size_t)e] = v;
            for (size_t d = idx.size(); d-- > 0;) { if (++idx[d] < t.shape[d]) break; idx[d] = 0; }
        }
    }
    return true;
}

// state_dict names of oracle/forward_ref.HerroNet -> the tensors of the HB200W1 blob (tools/export_weights.py does the same in numpy)
bool ts_to_canonical(const TsModel& m, int heads_hint, TsDims& d, std::map<std::string, std::vector<float>>& T, std::string& err) {
    auto get = [&](const std::string& k) -> const TsTensor* {
        auto it = m.tensors.find(k);
        return it == m.tensors.end() ? nullptr : &it->second;
    };
    auto need = [&](const std::string& k, size_t rank) -> const TsTensor* {
        const TsTensor* t = get(k);
        if (!t) { err = "the archive has no parameter '" + k + "' (not the architecture this library implements: oracle/forward_ref.py)"; return nullptr; }
        if (t->shape.size() != rank) { err = "parameter '" + k + "' has an unexpected rank"; return nullptr; }
        return t;
    };
    const TsTensor* sw = need("stem.weight", 4);
    const TsTensor* sb = sw ? need("stem.bias", 1) : nullptr;
    if (!sw || !sb) return false;
    if (sw->shape[1] != 7 || sw->shape[3] != 1 || sb->shape[0] != sw->shape[0]) { err = "stem.weight must be [C, 7, K, 1]"; return false; }
    const int64_t C = sw->shape[0], K = sw->shape[2];
    std::vector<float> stem_w = sw->data, stem_b = sb->data;  // [C,7,K,1] is [C,7,K] as stored
    if (const TsTensor* g = get("stem_bn.weight")) {          // fold BatchNorm (eval mode, eps 1e-5)
        const TsTensor *bb = get("stem_bn.bias"), *mu = get("stem_bn.running_mean"), *var = get("stem_bn.running_var");
        if (!bb || !mu || !var || (int64_t)g->data.size() != C || (int64_t)bb->data.size() != C || (int64_t)mu->data.size() != C || (int64_t)var->data.size() != C) {
            err = "incomplete stem_bn parameters";
            return false;
        }
        for (int64_t c = 0; c < C; c++) {
            const float s = g->data[c] / std::sqrt(var->data[c] + 1e-5f);
            for (int64_t i = 0; i < 7 * K; i++) stem_w[(size_t)(c * 7 * K + i)] *= s;
            stem_b[c] = (stem_b[c] - mu->data[c]) * s + bb->data[c];
        }
    }
    int layers = 0;
    while (get("layers." + std::to_string(layers) + ".qkv.weight")) layers++;
    const TsTensor *f1 = need("layers.0.ff1.weight", 2), *cw = f1 ? need("collapse.weight", 2) : nullptr;
    if (!f1 || !cw) return false;
    int heads = heads_hint;
    auto hi = m.ints.find("layers.0.H");
    if (hi != m.ints.end()) heads = (int)hi->second;
    d.stem_k = (int)K; d.channels = (int)C; d.heads = heads; d.layers = layers; d.ffn = (int)f1->shape[0]; d.collapse = (int)cw->shape[0];
    auto put = [&](const std::string& dst, const std::string& src, size_t rank, size_t count) -> bool {
        const TsTensor* t = need(src, rank);
        if (!t) return false;
        if (t->data.size() != count) { err = "parameter '" + src + "' has " + std::to_string(t->data.size()) + " elements, expected " + std::to_string(count); return false; }
        T[dst] = t->data;
        return true;
    };
    const size_t Cs = (size_t)C, F = (size_t)d.ffn, D = (size_t)d.collapse;
    T["stem_w"] = stem_w;
    T["stem_b"] = stem_b;
    if (!put("emb", "embedding.weight", 2, 12 * 6) || !put("read_pos", "read_pos", 2, 31 * Cs)) return false;
    for (int l = 0; l < layers; l++) {
        const std::string p = "layers." + std::to_string(l) + ".", q = "l" + std::to_string(l) + ".";
        if (!put(q + "ln1_g", p + "ln1.weight", 1, Cs) || !put(q + "ln1_b", p + "ln1.bias", 1, Cs) || !put(q + "wqkv", p + "qkv.weight", 2, 3 * Cs * Cs) ||
            !put(q + "bqkv", p + "qkv.bias", 1, 3 * Cs) || !put(q + "wo", p + "out.weight", 2, Cs * Cs) || !put(q + "bo", p + "out.bias", 1, Cs) ||
            !put(q + "ln2_g", p + "ln2.weight", 1, Cs) || !put(q + "ln2_b", p + "ln2.bias", 1, Cs) || !put(q + "w1", p + "ff1.weight", 2, F * Cs) ||
            !put(q + "b1", p + "ff1.bias", 1, F) || !put(q + "w2", p + "ff2.weight", 2, Cs * F) || !put(q + "b2", p + "ff2.bias", 1, Cs))
            return false;
    }
    if (!(put("lnf_g", "lnf.weight", 1, Cs) && put("lnf_b", "lnf.bias", 1, Cs) && put("wc", "collapse.weight", 2, D * 31 * Cs) && put("bc", "collapse.bias", 1, D) &&
          put("wb", "base_head.weight", 2, 5 * D) && put("bb", "base_head.bias", 1, 5) && put("wi", "info_head.weight", 2, D) && put("bi", "info_head.bias", 1, 1)))
        return false;
    // optional encoder stage across each window's supported positions (width D): pos_layers.{l}.*, head count pos_layers.0.H
    int pl = 0;
    while (get("pos_layers." + std::to_string(pl) + ".qkv.weight")) pl++;
    if (pl == 0) return true;
    auto ph = m.ints.find("pos_layers.0.H");
    if (ph == m.ints.end()) { err = "the archive has position layers but no head count 'pos_layers.0.H'"; return false; }
    const TsTensor* pf1 = need("pos_layers.0.ff1.weight", 2);
    if (!pf1) return false;
    d.pos_layers = pl; d.pos_heads = (int)ph->second; d.pos_ffn = (int)pf1->shape[0];
    const size_t P = (size_t)d.pos_ffn;
    for (int l = 0; l < pl; l++) {
        const std::string p = "pos_layers." + std::to_string(l) + ".", q = "p" + std::to_string(l) + ".";
        if (!put(q + "ln1_g", p + "ln1.weight", 1, D) || !put(q + "ln1_b", p + "ln1.bias", 1, D) || !put(q + "wqkv", p + "qkv.weight", 2, 3 * D * D) ||
            !put(q + "bqkv", p + "qkv.bias", 1, 3 * D) || !put(q + "wo", p + "out.weight", 2, D * D) || !put(q + "bo", p + "out.bias", 1, D) ||
            !put(q + "ln2_g", p + "ln2.weight", 1, D) || !put(q + "ln2_b", p + "ln2.bias", 1, D) || !put(q + "w1", p + "ff1.weight", 2, P * D) ||
            !put(q + "b1", p + "ff1.bias", 1, P) || !put(q + "w2", p + "ff2.weight", 2, D * P) || !put(q + "b2", p + "ff2.bias", 1, D))
            return false;
    }
    return true;
}

}  // namespace hb
