// align_oracle.cpp — test infrastructure: the sequential restatement of hb_align_overlaps' alignment (DESIGN.md §12), which the
// device must equal byte for byte.  Built with g++ into tests/_tmp on first use (tests/align_oracle.py); never linked into the
// product.
//
// Per overlap: T = target slice (forward), Q = query slice (reverse-complemented on strand 1), both as 2-bit codes.  Banded
// two-piece Gotoh (match +2, mismatch -4, gap cost min(4 + 2l, 24 + l)); row i holds columns c(i) - w <= j < c(i) + w with
// c(i) = floor(i m / n); traceback from (n, m); fix_cigar (left-align indels flanked by matches, drop a leading gap op, merge);
// end gaps trimmed into the coordinate shifts; identical base pairs inside M counted.
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

namespace {

constexpr int32_t NEG = -(1 << 30);
constexpr int OP_M = 0, OP_I = 1, OP_D = 2;
constexpr int32_t MATCH = 2, MISMATCH = -4, Q1 = 4, E1 = 2, Q2 = 24, E2 = 1;

struct Op { int kind; uint32_t len; };

inline int32_t clampv(int64_t v) { return v < NEG ? NEG : (int32_t)v; }

// fix_cigar (the reference's src/aligners.rs fix_cigar, restated): returns (tshift, qshift)
void fix_cigar(std::vector<Op>& c, const uint8_t* T, const uint8_t* Q, uint32_t& tshift, uint32_t& qshift) {
    size_t tpos = 0, qpos = 0;
    for (size_t i = 0; i < c.size(); i++) {
        if (c[i].kind == OP_M) { tpos += c[i].len; qpos += c[i].len; continue; }
        if (i > 0 && i + 1 < c.size() && c[i - 1].kind == OP_M && c[i + 1].kind == OP_M) {
            const size_t prev = c[i - 1].len, len = c[i].len;
            size_t l = 0;
            if (c[i].kind == OP_I) { while (l < prev && Q[qpos - 1 - l] == Q[qpos + len - 1 - l]) l++; }
            else { while (l < prev && T[tpos - 1 - l] == T[tpos + len - 1 - l]) l++; }
            if (l) { c[i - 1].len -= (uint32_t)l; c[i + 1].len += (uint32_t)l; tpos -= l; qpos -= l; }
        }
        if (c[i].kind == OP_I) qpos += c[i].len; else tpos += c[i].len;
    }
    tshift = qshift = 0;
    std::vector<Op> r;
    bool start = true;
    for (const Op& o : c) {
        if (start) {
            if (o.kind == OP_M) { if (o.len == 0) continue; start = false; r.push_back(o); continue; }
            start = false;
            (o.kind == OP_I ? qshift : tshift) = o.len;
            continue;
        }
        if (o.len) r.push_back(o);
    }
    c.clear();
    for (const Op& o : r) {
        if (!c.empty() && c.back().kind == o.kind) c.back().len += o.len;
        else c.push_back(o);
    }
}

std::string to_text(const std::vector<Op>& c) {
    std::string s;
    for (const Op& o : c) s += std::to_string(o.len) + "MID"[o.kind];
    return s;
}

bool parse(const char* s, std::vector<Op>& c) {
    c.clear();
    uint64_t v = 0;
    bool dig = false;
    for (; *s; s++) {
        if (*s >= '0' && *s <= '9') { v = v * 10 + (uint64_t)(*s - '0'); dig = true; continue; }
        const char* k = strchr("MID", *s);
        if (!k || !dig) return false;
        c.push_back(Op{(int)(k - "MID"), (uint32_t)v});
        v = 0;
        dig = false;
    }
    return !dig;
}

}  // namespace

extern "C" {

// fix_cigar on a text CIGAR over T / Q (ASCII or codes: compared for equality only).  out: the fixed CIGAR (NUL-terminated, cap
// bytes); shifts[0] = tshift, shifts[1] = qshift.  -> 0, or -1 for a malformed CIGAR or a too small buffer.
int ao_fix_cigar(const uint8_t* T, const uint8_t* Q, const char* cigar, char* out, uint32_t cap, uint32_t* shifts) {
    std::vector<Op> c;
    if (!parse(cigar, c)) return -1;
    fix_cigar(c, T, Q, shifts[0], shifts[1]);
    const std::string s = to_text(c);
    if (s.size() + 1 > cap) return -1;
    memcpy(out, s.c_str(), s.size() + 1);
    return 0;
}

// The alignment of T[0, n) and Q[0, m) (2-bit codes) in a band of 2w cells per row (n, m >= 1, m <= 2n, n <= 2m).
// res[0] = optimal score, res[1] = leading D, res[2] = leading I, res[3] = trailing D, res[4] = trailing I, res[5] = band edge
// (0 / 1), res[6] = identical pairs in M.  cigar: NUL-terminated final CIGAR (cap bytes).  -> 0, or -1 if cap is too small.
int ao_align(const uint8_t* T, uint32_t n, const uint8_t* Q, uint32_t m, uint32_t w, int32_t* res, char* cigar, uint32_t cap) {
    const int64_t W2 = 2 * (int64_t)w;
    auto cen = [&](int64_t i) { return (int64_t)(((uint64_t)i * m) / n); };
    std::vector<int32_t> pH(W2, NEG), pF1(W2, NEG), pF2(W2, NEG), H(W2), F1v(W2), F2v(W2), E1v(W2), E2v(W2);
    std::vector<uint8_t> tb((size_t)(n + 1) * W2, 0);
    int64_t plo = 0;
    for (int64_t i = 0; i <= (int64_t)n; i++) {
        const int64_t lo = cen(i) - w;
        for (int64_t k = 0; k < W2; k++) {
            const int64_t j = lo + k;
            if (j < 0 || j > (int64_t)m) { H[k] = F1v[k] = F2v[k] = E1v[k] = E2v[k] = NEG; continue; }
            int32_t upH = NEG, upF1 = NEG, upF2 = NEG, dgH = NEG;
            if (i > 0) {
                const int64_t ku = j - plo, kd = j - 1 - plo;
                if (ku >= 0 && ku < W2) { upH = pH[ku]; upF1 = pF1[ku]; upF2 = pF2[ku]; }
                if (j > 0 && kd >= 0 && kd < W2) dgH = pH[kd];
            }
            const int32_t lH = k ? H[k - 1] : NEG, lE1 = k ? E1v[k - 1] : NEG, lE2 = k ? E2v[k - 1] : NEG;
            uint8_t b = 0;
            int32_t o, x;
            o = clampv((int64_t)upH - Q1 - E1); x = clampv((int64_t)upF1 - E1);
            F1v[k] = x >= o ? x : o; b |= (x >= o) << 3;
            o = clampv((int64_t)upH - Q2 - E2); x = clampv((int64_t)upF2 - E2);
            F2v[k] = x >= o ? x : o; b |= (x >= o) << 4;
            o = clampv((int64_t)lH - Q1 - E1); x = clampv((int64_t)lE1 - E1);
            E1v[k] = x >= o ? x : o; b |= (x >= o) << 5;
            o = clampv((int64_t)lH - Q2 - E2); x = clampv((int64_t)lE2 - E2);
            E2v[k] = x >= o ? x : o; b |= (x >= o) << 6;
            int32_t h = NEG;
            int src = 0;
            if (i > 0 && j > 0) h = clampv((int64_t)dgH + (T[i - 1] == Q[j - 1] ? MATCH : MISMATCH));
            if (F1v[k] > h) { h = F1v[k]; src = 1; }
            if (F2v[k] > h) { h = F2v[k]; src = 2; }
            if (E1v[k] > h) { h = E1v[k]; src = 3; }
            if (E2v[k] > h) { h = E2v[k]; src = 4; }
            if (i == 0 && j == 0) { h = 0; src = 0; }
            H[k] = h;
            tb[(size_t)i * W2 + k] = (uint8_t)(b | src);
        }
        std::swap(pH, H); std::swap(pF1, F1v); std::swap(pF2, F2v);
        plo = lo;
    }
    res[0] = pH[(int64_t)m - (cen(n) - w)];
    // traceback
    std::vector<Op> rev;
    auto push = [&](int kind) { if (!rev.empty() && rev.back().kind == kind) rev.back().len++; else rev.push_back(Op{kind, 1}); };
    int64_t i = n, j = m;
    int st = 0;  // 0 H, 1 F1, 2 F2, 3 E1, 4 E2
    bool edge = false;
    while (i > 0 || j > 0 || st != 0) {
        const int64_t k = j - (cen(i) - w);
        if (i < 0 || j < 0 || k < 0 || k >= W2) return -2;
        if (k == 0 || k == W2 - 1) edge = true;
        const uint8_t b = tb[(size_t)i * W2 + k];
        switch (st) {
            case 0: { const int s = b & 7; if (s == 0) { push(OP_M); i--; j--; } else st = s; break; }
            case 1: push(OP_D); i--; st = (b >> 3 & 1) ? 1 : 0; break;
            case 2: push(OP_D); i--; st = (b >> 4 & 1) ? 2 : 0; break;
            case 3: push(OP_I); j--; st = (b >> 5 & 1) ? 3 : 0; break;
            case 4: push(OP_I); j--; st = (b >> 6 & 1) ? 4 : 0; break;
        }
    }
    std::vector<Op> c(rev.rbegin(), rev.rend());
    uint32_t ts = 0, qs = 0;
    fix_cigar(c, T, Q, ts, qs);
    uint32_t td = 0, ti = 0;
    while (!c.empty() && c.front().kind != OP_M) { (c.front().kind == OP_I ? qs : ts) += c.front().len; c.erase(c.begin()); }
    while (!c.empty() && c.back().kind != OP_M) { (c.back().kind == OP_I ? ti : td) += c.back().len; c.pop_back(); }
    uint32_t matches = 0;
    uint64_t t = ts, q = qs;
    for (const Op& o : c) {
        if (o.kind == OP_M) { for (uint32_t x = 0; x < o.len; x++) matches += T[t + x] == Q[q + x]; t += o.len; q += o.len; }
        else if (o.kind == OP_I) q += o.len;
        else t += o.len;
    }
    res[1] = (int32_t)ts; res[2] = (int32_t)qs; res[3] = (int32_t)td; res[4] = (int32_t)ti; res[5] = edge; res[6] = (int32_t)matches;
    const std::string s = to_text(c);
    if (s.size() + 1 > cap) return -1;
    memcpy(cigar, s.c_str(), s.size() + 1);
    return 0;
}

}  // extern "C"
