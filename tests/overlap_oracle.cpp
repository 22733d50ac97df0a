// overlap_oracle.cpp — test infrastructure: the sequential restatement of hb_find_overlaps (DESIGN.md §13), which the device
// must equal byte for byte.  Built with g++ into tests/_tmp on first use (tests/overlap_oracle.py); never linked into the
// product.  One loop per step of the definition: sketch, index and occurrence threshold, anchors, chain, strand choice, record.
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <map>
#include <tuple>
#include <vector>

namespace {

struct Params { uint32_t k, w, min_score, min_anchors, max_gap, bandwidth, max_iter, top_frac_ppm, min_occ; };

uint64_t hash64(uint64_t key, uint64_t mask) {
    key = (~key + (key << 21)) & mask;
    key = key ^ key >> 24;
    key = ((key + (key << 3)) + (key << 8)) & mask;
    key = key ^ key >> 14;
    key = ((key + (key << 2)) + (key << 4)) & mask;
    key = key ^ key >> 28;
    key = (key + (key << 31)) & mask;
    return key;
}

struct Mini { uint64_t h; uint32_t pos, z; };

std::vector<Mini> sketch(const uint8_t* c, uint32_t len, uint32_t k, uint32_t w) {
    const uint64_t mask = (k == 32) ? ~0ull : (1ull << (2 * k)) - 1;
    std::vector<Mini> km;  // the non-skipped k-mers, in position order
    for (uint32_t i = k - 1; i < len && len >= k; i++) {
        uint64_t f = 0, r = 0;
        for (uint32_t u = 0; u < k; u++) f = f << 2 | c[i - k + 1 + u];
        for (uint32_t u = 0; u < k; u++) r = r << 2 | (c[i - u] ^ 3u);
        if (f == r) continue;
        const uint64_t code = std::min(f, r);
        km.push_back(Mini{hash64(code, mask), i, r < f ? 1u : 0u});
    }
    std::vector<Mini> out;
    for (size_t e = w - 1; e < km.size(); e++) {
        size_t best = e + 1 - w;
        for (size_t b = e + 2 - w; b <= e; b++)
            if (km[b].h < km[best].h) best = b;  // leftmost on ties
        if (out.empty() || out.back().pos != km[best].pos) out.push_back(km[best]);
    }
    return out;
}

uint32_t max_occ_of(std::vector<uint32_t> occ, uint32_t top_frac_ppm, uint32_t min_occ) {
    if (occ.empty()) return min_occ;
    std::sort(occ.begin(), occ.end());
    const uint64_t nd = occ.size();
    const uint64_t rank = std::min<uint64_t>((1000000ull - top_frac_ppm) * nd / 1000000ull, nd - 1);
    return std::max(min_occ, occ[rank]);
}

uint32_t gap_cost(uint32_t l, uint32_t k) {
    if (l == 0) return 0;
    uint32_t lg = 0;
    while ((l >> (lg + 1)) != 0) lg++;
    return (uint32_t)((uint64_t)k * l / 100) + lg / 2;
}

struct Chain { int64_t score; uint32_t n_anchors, first, last, covered; };

// anchors (x[], y[]) of one group, sorted by (x, y)
Chain chain(const uint32_t* x, const uint32_t* y, uint32_t n, const Params& p) {
    std::vector<int64_t> f(n);
    std::vector<int64_t> pred(n, -1);
    for (uint32_t a = 0; a < n; a++) {
        f[a] = p.k;
        const int64_t lo = std::max<int64_t>(0, (int64_t)a - p.max_iter);
        for (int64_t b = (int64_t)a - 1; b >= lo; b--) {
            const int64_t dx = (int64_t)x[a] - x[b];
            if (dx > p.max_gap) break;
            const int64_t dy = (int64_t)y[a] - y[b];
            if (dx <= 0 || dy <= 0 || dy > p.max_gap) continue;
            const int64_t l = dx > dy ? dx - dy : dy - dx;
            if (l > p.bandwidth) continue;
            const int64_t sc = f[b] + std::min<int64_t>(std::min(dx, dy), p.k) - gap_cost((uint32_t)l, p.k);
            if (sc > f[a]) { f[a] = sc; pred[a] = b; }
        }
    }
    Chain c{0, 0, 0, 0, 0};
    if (!n) return c;
    uint32_t end = 0;
    for (uint32_t a = 1; a < n; a++) if (f[a] > f[end]) end = a;
    c.score = f[end];
    c.last = end;
    int64_t cov_lo = -1;  // the union of the chain's k-mers [x - k + 1, x], walked from the last anchor down
    for (int64_t a = end; a >= 0; a = pred[a]) {
        c.n_anchors++;
        c.first = (uint32_t)a;
        const int64_t s = (int64_t)x[a] - p.k + 1, e = (int64_t)x[a] + 1;
        if (cov_lo < 0) { c.covered += (uint32_t)(e - s); cov_lo = s; }
        else if (e <= cov_lo) { c.covered += (uint32_t)(e - s); cov_lo = s; }
        else if (s < cov_lo) { c.covered += (uint32_t)(cov_lo - s); cov_lo = s; }
    }
    return c;
}

struct Rec { uint32_t qid, qlen, qstart, qend, strand, tid, tlen, tstart, tend, score, n_anchors, covered; };

}  // namespace

extern "C" {

uint64_t oo_hash64(uint64_t key, uint64_t mask) { return hash64(key, mask); }

// A read's minimizers (codes c[len]): writes at most cap of them; returns how many there are
uint32_t oo_sketch(const uint8_t* c, uint32_t len, uint32_t k, uint32_t w, uint64_t* h, uint32_t* pos, uint32_t* z, uint32_t cap) {
    const std::vector<Mini> m = sketch(c, len, k, w);
    for (size_t i = 0; i < m.size() && i < cap; i++) { h[i] = m[i].h; pos[i] = m[i].pos; z[i] = m[i].z; }
    return (uint32_t)m.size();
}

uint32_t oo_max_occ(const uint32_t* occ, uint32_t n, uint32_t top_frac_ppm, uint32_t min_occ) {
    return max_occ_of(std::vector<uint32_t>(occ, occ + n), top_frac_ppm, min_occ);
}

// One group's chain: out = {score, n_anchors, first, last, covered}
void oo_chain(const uint32_t* x, const uint32_t* y, uint32_t n, const uint32_t* params, int64_t* out) {
    Params p;
    memcpy(&p, params, sizeof p);
    const Chain c = chain(x, y, n, p);
    out[0] = c.score; out[1] = c.n_anchors; out[2] = c.first; out[3] = c.last; out[4] = c.covered;
}

// The whole call: reads as codes (codes[off[r] .. off[r+1])), the call's targets, params (9 values, defaults applied by the
// caller).  Returns the number of records; writes at most cap of them as 12 u32 each (qid qlen qstart qend strand tid tlen
// tstart tend score n_anchors covered).  stats: max_occ, n_filtered_hashes, index_entries, query_minimizers, anchors.
uint64_t oo_find(const uint8_t* codes, const uint64_t* off, uint32_t n_reads, const uint32_t* targets, uint32_t n_targets,
                 const uint32_t* params, uint32_t* out, uint64_t cap, uint64_t* stats) {
    Params p;
    memcpy(&p, params, sizeof p);
    std::vector<std::vector<Mini>> sk(n_reads);
    for (uint32_t r = 0; r < n_reads; r++) sk[r] = sketch(codes + off[r], (uint32_t)(off[r + 1] - off[r]), p.k, p.w);
    // index and threshold
    std::map<uint64_t, std::vector<std::tuple<uint32_t, uint32_t, uint32_t>>> index;  // h -> (target in call, i, z)
    uint64_t entries = 0;
    for (uint32_t t = 0; t < n_targets; t++)
        for (const Mini& m : sk[targets[t]]) { index[m.h].emplace_back(t, m.pos, m.z); entries++; }
    std::vector<uint32_t> occ;
    for (auto& kv : index) occ.push_back((uint32_t)kv.second.size());
    const uint32_t max_occ = max_occ_of(occ, p.top_frac_ppm, p.min_occ);
    uint64_t n_filtered = 0;
    for (uint32_t o : occ) n_filtered += o > max_occ;
    // anchors per group (t, q, s), then chains
    std::vector<Rec> recs;
    uint64_t qmin = 0, n_anchors = 0;
    for (uint32_t q = 0; q < n_reads; q++) {
        const uint32_t qlen = (uint32_t)(off[q + 1] - off[q]);
        qmin += sk[q].size();
        std::map<std::tuple<uint32_t, uint32_t>, std::vector<std::pair<uint32_t, uint32_t>>> groups;  // (t, s) -> (x, y)
        for (const Mini& m : sk[q]) {
            auto it = index.find(m.h);
            if (it == index.end() || it->second.size() > max_occ) continue;
            for (auto& [t, i, zt] : it->second) {
                if (targets[t] == q) continue;
                const uint32_t s = m.z ^ zt;
                const uint32_t y = s ? qlen + p.k - 2 - m.pos : m.pos;
                groups[{t, s}].emplace_back(i, y);
                n_anchors++;
            }
        }
        for (auto& kv : groups) std::sort(kv.second.begin(), kv.second.end());
        for (uint32_t t = 0; t < n_targets; t++) {
            bool have = false;
            Rec best{};
            for (uint32_t s = 0; s < 2; s++) {
                auto it = groups.find({t, s});
                if (it == groups.end()) continue;
                const auto& a = it->second;
                const uint32_t n = (uint32_t)a.size();
                std::vector<uint32_t> x(n), y(n);
                for (uint32_t j = 0; j < n; j++) { x[j] = a[j].first; y[j] = a[j].second; }
                const Chain c = chain(x.data(), y.data(), n, p);
                if (c.score < p.min_score || c.n_anchors < p.min_anchors) continue;
                if (have && c.score <= best.score) continue;
                const uint32_t tr = targets[t];
                Rec r{q, qlen, 0, 0, s, tr, (uint32_t)(off[tr + 1] - off[tr]), x[c.first] - p.k + 1, x[c.last] + 1,
                      (uint32_t)c.score, c.n_anchors, c.covered};
                if (s == 0) { r.qstart = y[c.first] - p.k + 1; r.qend = y[c.last] + 1; }
                else { r.qstart = qlen - y[c.last] - 1; r.qend = qlen - y[c.first] + p.k - 1; }
                best = r;
                have = true;
            }
            if (have) recs.push_back(best);
        }
    }
    // built in ascending qid; the stable sort puts them in call-target order
    std::vector<uint32_t> tpos(n_reads, 0);
    for (uint32_t t = 0; t < n_targets; t++) tpos[targets[t]] = t;
    std::stable_sort(recs.begin(), recs.end(), [&](const Rec& a, const Rec& b) { return tpos[a.tid] < tpos[b.tid]; });
    for (size_t i = 0; i < recs.size() && i < cap; i++) memcpy(out + 12 * i, &recs[i], 48);
    stats[0] = max_occ; stats[1] = n_filtered; stats[2] = entries; stats[3] = qmin; stats[4] = n_anchors;
    return recs.size();
}

}  // extern "C"
