// io.cpp — the host data plane around the hot path, natively and multi-threaded (SURVEY.md §8f-2, §8f-4):
//
//   hbh_reads_*    FASTQ (plain or .gz) -> read ids, descriptions, qualities, 2-bit packed sequences in the HAECSeq layout
//                  (haec_io::get_reads, src/haec_io.rs:37-75,121-136): reads shorter than the window are dropped (:48), the
//                  id is split from the description at the first space / tab (:52-54), cluster filter (:64-70)
//   hbh_alns_*     a `--read-alns` directory of *.oec.zst batches -> alignments grouped by target
//                  (overlaps::read_batches + parse_paf, src/overlaps.rs:288-323,117-202): header lines skipped, unknown read
//                  names skipped, core filter on the target, self overlaps dropped, only the first line of an ordered
//                  (query, target) pair per batch file kept.  The reference decodes and parses batch files one after the
//                  other on one thread; here every file is decompressed (libzstd through dlopen: the image ships the
//                  library but no header) and parsed by its own worker.
//   hbh_fasta_*    correction_writer / write_sequence (src/lib.rs:267-317): `>id[:k] description\n seq\n`
//   hbh_inference  the whole `herro inference --read-alns` pipeline over the public C ABI of libherro_b200: ingest ->
//                  hb_upload_reads (or one host read store for all devices) -> feature threads (hb_submit_alignments) -> consumer (hb_poll_corrected) -> FASTA,
//                  with the time of every stage reported.
//
// In the deployed layout these stay in the Rust host; they exist here because no Rust toolchain is available offline and
// because, once the GPU path runs at hundreds of Mbases/s, single-threaded ingest is the bottleneck (SURVEY.md §8f).
#include <dirent.h>
#include <dlfcn.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <fcntl.h>
#include <unistd.h>
#include <zlib.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <string>
#include <string_view>
#include <thread>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "../../include/herro_b200.h"

namespace {

double now_s() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

thread_local std::string t_err;

// ---------------------------------------------------------------------------------------------- file -> memory
struct FileBytes {
    std::vector<uint8_t> owned;  // gz-inflated contents
    const uint8_t* p = nullptr;
    size_t n = 0;
    void* map = nullptr;
    size_t map_len = 0;
    ~FileBytes() { if (map) munmap(map, map_len); }
};

bool load_file(const std::string& path, FileBytes& fb) {
    int fd = open(path.c_str(), O_RDONLY);
    if (fd < 0) { t_err = "cannot open " + path; return false; }
    struct stat st;
    if (fstat(fd, &st) != 0) { close(fd); t_err = "cannot stat " + path; return false; }
    unsigned char magic[2] = {0, 0};
    const bool gz = st.st_size >= 2 && pread(fd, magic, 2, 0) == 2 && magic[0] == 0x1f && magic[1] == 0x8b;
    if (gz) {
        close(fd);
        gzFile g = gzopen(path.c_str(), "rb");
        if (!g) { t_err = "cannot gzopen " + path; return false; }
        gzbuffer(g, 1 << 20);
        std::vector<uint8_t>& o = fb.owned;
        size_t cap = std::max<size_t>((size_t)st.st_size * 4, 1 << 20);
        o.resize(cap);
        size_t n = 0;
        for (;;) {
            if (n == o.size()) o.resize(o.size() * 2);
            const int r = gzread(g, o.data() + n, (unsigned)std::min<size_t>(o.size() - n, 1u << 30));
            if (r < 0) { gzclose(g); t_err = "gzip error in " + path; return false; }
            if (r == 0) break;
            n += (size_t)r;
        }
        gzclose(g);
        o.resize(n);
        fb.p = o.data();
        fb.n = n;
        return true;
    }
    if (st.st_size == 0) { close(fd); fb.p = nullptr; fb.n = 0; return true; }
    void* m = mmap(nullptr, (size_t)st.st_size, PROT_READ, MAP_PRIVATE, fd, 0);
    close(fd);
    if (m == MAP_FAILED) { t_err = "cannot mmap " + path; return false; }
    madvise(m, (size_t)st.st_size, MADV_SEQUENTIAL);
    fb.map = m; fb.map_len = (size_t)st.st_size;
    fb.p = (const uint8_t*)m; fb.n = (size_t)st.st_size;
    return true;
}

// ---------------------------------------------------------------------------------------------- zstd through dlopen
struct ZInBuf { const void* src; size_t size; size_t pos; };
struct ZOutBuf { void* dst; size_t size; size_t pos; };
struct Zstd {
    void* h = nullptr;
    void* (*createDStream)() = nullptr;
    size_t (*freeDStream)(void*) = nullptr;
    size_t (*initDStream)(void*) = nullptr;
    size_t (*decompressStream)(void*, ZOutBuf*, ZInBuf*) = nullptr;
    unsigned (*isError)(size_t) = nullptr;
    unsigned long long (*getFrameContentSize)(const void*, size_t) = nullptr;
    bool ok = false;
};
const Zstd& zstd() {
    static Zstd z = [] {
        Zstd r;
        for (const char* name : {"libzstd.so.1", "libzstd.so"}) {
            r.h = dlopen(name, RTLD_NOW | RTLD_GLOBAL);
            if (r.h) break;
        }
        if (!r.h) return r;
        r.createDStream = (void* (*)())dlsym(r.h, "ZSTD_createDStream");
        r.freeDStream = (size_t(*)(void*))dlsym(r.h, "ZSTD_freeDStream");
        r.initDStream = (size_t(*)(void*))dlsym(r.h, "ZSTD_initDStream");
        r.decompressStream = (size_t(*)(void*, ZOutBuf*, ZInBuf*))dlsym(r.h, "ZSTD_decompressStream");
        r.isError = (unsigned (*)(size_t))dlsym(r.h, "ZSTD_isError");
        r.getFrameContentSize = (unsigned long long (*)(const void*, size_t))dlsym(r.h, "ZSTD_getFrameContentSize");
        r.ok = r.createDStream && r.freeDStream && r.initDStream && r.decompressStream && r.isError;
        return r;
    }();
    return z;
}

bool zstd_decompress(const uint8_t* src, size_t n, std::vector<uint8_t>& out) {
    const Zstd& z = zstd();
    if (!z.ok) { t_err = "libzstd.so.1 not found"; return false; }
    void* ds = z.createDStream();
    if (!ds) { t_err = "ZSTD_createDStream failed"; return false; }
    z.initDStream(ds);
    size_t guess = n * 6 + (1 << 16);
    if (z.getFrameContentSize) {
        const unsigned long long cs = z.getFrameContentSize(src, n);
        if (cs != 0ull - 1 && cs != 0ull - 2 && cs > 0) guess = (size_t)cs;
    }
    out.resize(guess);
    ZInBuf in{src, n, 0};
    size_t produced = 0;
    for (;;) {
        if (produced == out.size()) out.resize(out.size() * 2);
        ZOutBuf ob{out.data() + produced, out.size() - produced, 0};
        const size_t r = z.decompressStream(ds, &ob, &in);
        produced += ob.pos;
        if (z.isError(r)) { z.freeDStream(ds); t_err = "zstd stream error"; return false; }
        if (in.pos == in.size && ob.pos < ob.size) break;  // input consumed and the output buffer was not the limit
    }
    z.freeDStream(ds);
    out.resize(produced);
    return true;
}

inline const uint8_t* find_nl(const uint8_t* p, const uint8_t* e) {
    const void* q = memchr(p, '\n', (size_t)(e - p));
    return q ? (const uint8_t*)q : e;
}

}  // namespace

// ================================================================================================ reads
struct hbh_reads {
    std::vector<std::string> id, desc;
    std::vector<uint8_t> has_desc;
    std::vector<uint32_t> len;
    std::vector<uint64_t> woff, qoff;       // [n+1]
    std::vector<uint64_t> words;            // 2-bit packed, all reads
    std::vector<uint8_t> qual;              // all reads
    std::vector<const uint64_t*> word_ptr;  // per read, for hb_upload_reads
    std::vector<const uint8_t*> qual_ptr;
    std::vector<const char*> name_ptr;      // NUL-terminated ids
    std::unordered_map<std::string_view, uint32_t> name_to_id;
    double t_load = 0, t_pack = 0;
    uint64_t skipped_short = 0;
};

struct hbh_alns {
    std::vector<std::vector<uint8_t>> text;  // decompressed batch files (the CIGARs point into them)
    std::vector<hb_overlap> ovl;             // grouped by target
    std::vector<uint32_t> tgt_rid;
    std::vector<uint64_t> tgt_off;           // [n_targets+1] into ovl
    double t_decode = 0, t_parse = 0;
    uint64_t lines = 0, kept = 0, compressed_bytes = 0, text_bytes = 0;
    uint32_t files = 0;
};

struct hbh_fasta {
    FILE* f = nullptr;
    std::mutex mu;
    uint64_t records = 0, bases = 0;
};

extern "C" {

const char* hbh_last_error() { return t_err.c_str(); }

// `path`: a FASTQ file (plain or gzip) or a directory holding *.fastq / *.fastq.gz (src/lib.rs:241-265).  core / neighbour:
// read ids of a cluster file (src/lib.rs:208-239), or NULL / 0 for no filter.
int hbh_reads_load(const char* path, uint32_t min_len, const char* const* core, uint32_t n_core, const char* const* neighbour,
                   uint32_t n_neigh, int threads, hbh_reads** out) {
    if (!path || !out) return HB_ERR_ARG;
    *out = nullptr;
    const double t0 = now_s();
    std::vector<std::string> files;
    struct stat st;
    if (stat(path, &st) != 0) { t_err = std::string("cannot stat ") + path; return HB_ERR_ARG; }
    if (S_ISDIR(st.st_mode)) {
        DIR* d = opendir(path);
        if (!d) { t_err = std::string("cannot open directory ") + path; return HB_ERR_ARG; }
        while (dirent* e = readdir(d)) {
            const std::string nme = e->d_name;
            auto ends = [&](const char* suf) { const size_t l = strlen(suf); return nme.size() >= l && nme.compare(nme.size() - l, l, suf) == 0; };
            if (ends(".fastq") || ends(".fastq.gz")) files.push_back(std::string(path) + "/" + nme);
        }
        closedir(d);
        std::sort(files.begin(), files.end());
    } else {
        files.push_back(path);
    }
    const bool filter = core && neighbour;
    std::unordered_set<std::string_view> keep;
    if (filter) {
        for (uint32_t i = 0; i < n_core; i++) keep.insert(core[i]);
        for (uint32_t i = 0; i < n_neigh; i++) keep.insert(neighbour[i]);
    }
    auto* R = new hbh_reads();
    struct Rec { const uint8_t *hdr, *hdr_end, *seq, *qual; uint32_t len; };
    std::vector<FileBytes> bytes(files.size());
    std::vector<Rec> recs;
    for (size_t fi = 0; fi < files.size(); fi++) {
        if (!load_file(files[fi], bytes[fi])) { delete R; return HB_ERR_ARG; }
        const uint8_t *p = bytes[fi].p, *e = p + bytes[fi].n;
        while (p < e) {
            if (*p == '\n' || *p == '\r') { p++; continue; }
            if (*p != '@') { t_err = "not a FASTQ record (qualities must be present) in " + files[fi]; delete R; return HB_ERR_INPUT; }
            const uint8_t* h_end = find_nl(p, e);
            const uint8_t* s = h_end + 1;
            if (s >= e) break;
            const uint8_t* s_end = find_nl(s, e);
            const uint8_t* plus = s_end + 1;
            if (plus >= e || *plus != '+') { t_err = "multi-line or truncated FASTQ record in " + files[fi]; delete R; return HB_ERR_INPUT; }
            const uint8_t* q = find_nl(plus, e) + 1;
            if (q > e) q = e;
            const uint8_t* q_end = find_nl(q, e);
            size_t sl = (size_t)(s_end - s), ql = (size_t)(q_end - q);
            if (sl && s[sl - 1] == '\r') sl--;
            if (ql && q[ql - 1] == '\r') ql--;
            if (sl != ql) { t_err = "sequence / quality length mismatch in " + files[fi]; delete R; return HB_ERR_INPUT; }
            const uint8_t* he = h_end;
            if (he > p && he[-1] == '\r') he--;
            if (sl >= min_len) {  // src/haec_io.rs:48
                bool take = true;
                if (filter) {
                    const uint8_t* ie = p + 1;
                    while (ie < he && *ie != ' ' && *ie != '\t') ie++;
                    take = keep.count(std::string_view((const char*)p + 1, (size_t)(ie - p - 1))) != 0;
                }
                if (take) recs.push_back(Rec{p + 1, he, s, q, (uint32_t)sl});
            } else {
                R->skipped_short++;
            }
            p = q_end + 1;
        }
    }
    const uint32_t n = (uint32_t)recs.size();
    R->id.resize(n); R->desc.resize(n); R->has_desc.assign(n, 0); R->len.resize(n);
    R->woff.assign(n + 1, 0); R->qoff.assign(n + 1, 0);
    for (uint32_t i = 0; i < n; i++) {
        const Rec& r = recs[i];
        const uint8_t* ie = r.hdr;
        while (ie < r.hdr_end && *ie != ' ' && *ie != '\t') ie++;
        R->id[i].assign((const char*)r.hdr, (size_t)(ie - r.hdr));
        if (ie < r.hdr_end) { R->has_desc[i] = 1; R->desc[i].assign((const char*)ie + 1, (size_t)(r.hdr_end - ie - 1)); }
        R->len[i] = r.len;
        R->woff[i + 1] = R->woff[i] + (r.len + 31) / 32;
        R->qoff[i + 1] = R->qoff[i] + r.len;
    }
    R->t_load = now_s() - t0;
    const double t1 = now_s();
    R->words.assign(R->woff[n] + 1, 0);
    R->qual.resize(R->qoff[n]);
    static const auto lut = [] {
        std::vector<uint8_t> t(256, 255);
        t['A'] = t['a'] = 0; t['C'] = t['c'] = 1; t['G'] = t['g'] = 2; t['T'] = t['t'] = 3;
        return t;
    }();
    std::atomic<uint32_t> next{0};
    std::atomic<int> bad{0};
    auto work = [&]() {
        for (;;) {
            const uint32_t i0 = next.fetch_add(32);
            if (i0 >= n) break;
            for (uint32_t i = i0; i < std::min(n, i0 + 32); i++) {
                const Rec& r = recs[i];
                uint64_t* w = R->words.data() + R->woff[i];
                for (uint32_t b = 0; b < r.len; b += 32) {
                    const uint32_t m = std::min<uint32_t>(32, r.len - b);
                    uint64_t v = 0;
                    uint8_t any = 0;
                    for (uint32_t k = 0; k < m; k++) { const uint8_t c = lut[r.seq[b + k]]; any |= c; v |= (uint64_t)(c & 3) << (2 * k); }
                    if (any > 3) bad = 1;
                    w[b >> 5] = v;
                }
                memcpy(R->qual.data() + R->qoff[i], r.qual, r.len);
            }
        }
    };
    std::vector<std::thread> th;
    for (int i = 0; i < std::max(1, threads); i++) th.emplace_back(work);
    for (auto& t : th) t.join();
    if (bad.load()) { t_err = "non-ACGT base: the reference's 2-bit packing is undefined for it (SURVEY.md H12)"; delete R; return HB_ERR_INPUT; }
    R->word_ptr.resize(n); R->qual_ptr.resize(n); R->name_ptr.resize(n);
    R->name_to_id.reserve((size_t)n * 2);
    for (uint32_t i = 0; i < n; i++) {
        R->word_ptr[i] = R->words.data() + R->woff[i];
        R->qual_ptr[i] = R->qual.data() + R->qoff[i];
        R->name_ptr[i] = R->id[i].c_str();
        R->name_to_id.emplace(std::string_view(R->id[i]), i);  // a repeated id keeps its first index
    }
    R->t_pack = now_s() - t1;
    *out = R;
    return HB_OK;
}

void hbh_reads_free(hbh_reads* r) { delete r; }
uint32_t hbh_reads_count(const hbh_reads* r) { return r ? (uint32_t)r->id.size() : 0; }
const uint32_t* hbh_reads_lens(const hbh_reads* r) { return r->len.data(); }
const uint64_t* const* hbh_reads_word_ptrs(const hbh_reads* r) { return r->word_ptr.data(); }
const uint8_t* const* hbh_reads_qual_ptrs(const hbh_reads* r) { return r->qual_ptr.data(); }
const char* const* hbh_reads_names(const hbh_reads* r) { return r->name_ptr.data(); }
const char* hbh_reads_description(const hbh_reads* r, uint32_t i) { return r->has_desc[i] ? r->desc[i].c_str() : nullptr; }
// stats4: load seconds (read + scan), pack seconds, reads dropped as shorter than min_len, total bases
void hbh_reads_stats(const hbh_reads* r, double* stats4) {
    stats4[0] = r->t_load; stats4[1] = r->t_pack; stats4[2] = (double)r->skipped_short; stats4[3] = (double)r->qoff.back();
}

// ================================================================================================ alignments
namespace {
struct FileAlns {
    std::vector<hb_overlap> ovl;  // in file order
    std::vector<uint32_t> order;  // target of first appearance order
    uint64_t lines = 0;
    double t_decode = 0, t_parse = 0;
    bool ok = true;
    std::string err;
};

inline bool parse_u32(const uint8_t* p, const uint8_t* e, uint32_t& v) {  // bytes_to_u32: decimal digits only
    uint64_t x = 0;
    if (p == e) return false;
    for (; p < e; p++) {
        if (*p < '0' || *p > '9') return false;
        x = x * 10 + (*p - '0');
        if (x > 0xffffffffull) return false;
    }
    v = (uint32_t)x;
    return true;
}

void parse_batch(const hbh_reads* R, const std::unordered_set<std::string_view>* core, const std::vector<uint8_t>& text, FileAlns& fa) {
    const uint8_t *p = text.data(), *e = p + text.size();
    // header: <N>\n then N read ids (src/overlaps.rs:303-319)
    const uint8_t* nl = find_nl(p, e);
    uint32_t n_targets = 0;
    if (!parse_u32(p, nl, n_targets)) { fa.ok = false; fa.err = "bad batch header"; return; }
    p = nl + 1;
    for (uint32_t i = 0; i < n_targets && p < e; i++) p = find_nl(p, e) + 1;
    std::unordered_set<uint64_t> seen;
    while (p < e) {
        const uint8_t* le = find_nl(p, e);
        if (le == p) { p = le + 1; continue; }
        fa.lines++;
        const uint8_t* f[9][2];
        const uint8_t* c = p;
        int nf = 0;
        const uint8_t* last_b = p;
        while (c <= le && nf < 9) {
            const uint8_t* t = (const uint8_t*)memchr(c, '\t', (size_t)(le - c));
            if (!t) t = le;
            f[nf][0] = c; f[nf][1] = t;
            nf++;
            c = t + 1;
        }
        // the CIGAR is the LAST tab-separated field, minus its 5-byte tag "cg:Z:" (src/overlaps.rs:172)
        for (const uint8_t* t = le; t > p; t--) if (t[-1] == '\t') { last_b = t; break; }
        if (nf < 9 || last_b + 5 > le) { fa.ok = false; fa.err = "malformed PAF line"; return; }
        auto qit = R->name_to_id.find(std::string_view((const char*)f[0][0], (size_t)(f[0][1] - f[0][0])));
        if (qit == R->name_to_id.end()) { p = le + 1; continue; }
        hb_overlap o{};
        o.qid = qit->second;
        const std::string_view tname((const char*)f[5][0], (size_t)(f[5][1] - f[5][0]));
        if (!parse_u32(f[1][0], f[1][1], o.qlen) || !parse_u32(f[2][0], f[2][1], o.qstart) || !parse_u32(f[3][0], f[3][1], o.qend)) {
            fa.ok = false; fa.err = "malformed PAF number"; return;
        }
        const uint8_t sc = f[4][0] < f[4][1] ? *f[4][0] : 0;
        if (sc != '+' && sc != '-') { fa.ok = false; fa.err = "Invalid strand character."; return; }
        o.strand = sc == '-';
        if (core && !core->count(tname)) { p = le + 1; continue; }
        auto tit = R->name_to_id.find(tname);
        if (tit == R->name_to_id.end()) { p = le + 1; continue; }
        o.tid = tit->second;
        if (!parse_u32(f[6][0], f[6][1], o.tlen) || !parse_u32(f[7][0], f[7][1], o.tstart) || !parse_u32(f[8][0], f[8][1], o.tend)) {
            fa.ok = false; fa.err = "malformed PAF number"; return;
        }
        if (o.tid == o.qid) { p = le + 1; continue; }                                   // no self overlaps
        if (!seen.insert(((uint64_t)o.qid << 32) | o.tid).second) { p = le + 1; continue; }  // first overlap of a pair wins
        o.cigar = last_b + 5;
        o.cigar_len = (uint32_t)(le - (last_b + 5));
        if (o.cigar_len && o.cigar[o.cigar_len - 1] == '\r') o.cigar_len--;
        fa.ovl.push_back(o);
        p = le + 1;
    }
}
}  // namespace

int hbh_alns_load(const char* dir, const hbh_reads* reads, const char* const* core, uint32_t n_core, int threads, hbh_alns** out) {
    if (!dir || !reads || !out) return HB_ERR_ARG;
    *out = nullptr;
    std::vector<std::string> files;
    DIR* d = opendir(dir);
    if (!d) { t_err = std::string("cannot open directory ") + dir; return HB_ERR_ARG; }
    while (dirent* e = readdir(d)) {
        const std::string nme = e->d_name;
        if (nme.size() > 8 && nme.compare(nme.size() - 8, 8, ".oec.zst") == 0) files.push_back(std::string(dir) + "/" + nme);
    }
    closedir(d);
    std::sort(files.begin(), files.end());
    std::unordered_set<std::string_view> core_set;
    if (core) for (uint32_t i = 0; i < n_core; i++) core_set.insert(core[i]);
    auto* A = new hbh_alns();
    A->files = (uint32_t)files.size();
    A->text.resize(files.size());
    std::vector<FileAlns> per(files.size());
    std::atomic<uint32_t> next{0};
    std::atomic<uint64_t> comp{0};
    auto work = [&]() {
        for (;;) {
            const uint32_t i = next.fetch_add(1);
            if (i >= files.size()) break;
            FileAlns& fa = per[i];
            const double t0 = now_s();
            FileBytes fb;
            if (!load_file(files[i], fb)) { fa.ok = false; fa.err = t_err; continue; }
            comp.fetch_add(fb.n);
            if (!zstd_decompress(fb.p, fb.n, A->text[i])) { fa.ok = false; fa.err = t_err + " in " + files[i]; continue; }
            fa.t_decode = now_s() - t0;
            const double t1 = now_s();
            parse_batch(reads, core ? &core_set : nullptr, A->text[i], fa);
            fa.t_parse = now_s() - t1;
        }
    };
    std::vector<std::thread> th;
    for (int i = 0; i < std::max(1, std::min<int>(threads, (int)files.size())); i++) th.emplace_back(work);
    for (auto& t : th) t.join();
    // group by target inside every file, in order of first appearance (the reference's HashMap order is arbitrary, F8); a target
    // named in several files is sent once per file, like the reference's per-batch maps
    for (size_t i = 0; i < files.size(); i++) {
        FileAlns& fa = per[i];
        if (!fa.ok) { t_err = fa.err; delete A; return HB_ERR_INPUT; }
        A->t_decode += fa.t_decode; A->t_parse += fa.t_parse; A->lines += fa.lines; A->kept += fa.ovl.size();
        A->text_bytes += A->text[i].size();
        std::unordered_map<uint32_t, uint32_t> slot;
        std::vector<uint32_t> cnt;
        std::vector<uint32_t> tids;
        for (const hb_overlap& o : fa.ovl) {
            auto it = slot.find(o.tid);
            if (it == slot.end()) { slot.emplace(o.tid, (uint32_t)cnt.size()); cnt.push_back(1); tids.push_back(o.tid); }
            else cnt[it->second]++;
        }
        const size_t base = A->ovl.size();
        std::vector<uint64_t> start(cnt.size() + 1, 0);
        for (size_t k = 0; k < cnt.size(); k++) start[k + 1] = start[k] + cnt[k];
        A->ovl.resize(base + fa.ovl.size());
        std::vector<uint64_t> fill(start.begin(), start.end() - 1);
        for (const hb_overlap& o : fa.ovl) A->ovl[base + fill[slot[o.tid]]++] = o;
        for (size_t k = 0; k < cnt.size(); k++) {
            if (A->tgt_off.empty()) A->tgt_off.push_back(0);
            A->tgt_rid.push_back(tids[k]);
            A->tgt_off.push_back(base + start[k + 1]);
        }
    }
    if (A->tgt_off.empty()) A->tgt_off.push_back(0);
    A->compressed_bytes = comp.load();
    *out = A;
    return HB_OK;
}

void hbh_alns_free(hbh_alns* a) { delete a; }
uint32_t hbh_alns_targets(const hbh_alns* a) { return (uint32_t)a->tgt_rid.size(); }
const uint32_t* hbh_alns_target_rids(const hbh_alns* a) { return a->tgt_rid.data(); }
const uint64_t* hbh_alns_target_offsets(const hbh_alns* a) { return a->tgt_off.data(); }
const hb_overlap* hbh_alns_overlaps(const hbh_alns* a) { return a->ovl.data(); }
// stats6: sum of per-file decode seconds, sum of per-file parse seconds, PAF lines, alignments kept, compressed bytes, text bytes
void hbh_alns_stats(const hbh_alns* a, double* stats6) {
    stats6[0] = a->t_decode; stats6[1] = a->t_parse; stats6[2] = (double)a->lines; stats6[3] = (double)a->kept;
    stats6[4] = (double)a->compressed_bytes; stats6[5] = (double)a->text_bytes;
}

// ================================================================================================ FASTA
int hbh_fasta_open(const char* path, hbh_fasta** out) {
    if (!path || !out) return HB_ERR_ARG;
    FILE* f = fopen(path, "wb");
    if (!f) { t_err = std::string("cannot create ") + path; return HB_ERR_ARG; }
    setvbuf(f, nullptr, _IOFBF, 1 << 22);
    auto* w = new hbh_fasta();
    w->f = f;
    *out = w;
    return HB_OK;
}
// write_sequence (src/lib.rs:294-317): `>id` + (":k " when the read has several segments, " " otherwise) + description + "\n" + seq + "\n"
int hbh_fasta_write(hbh_fasta* w, const char* id, const char* description, const uint8_t* seqs, const uint32_t* seg_len, uint32_t n_segs) {
    if (!w || !id || (n_segs && (!seqs || !seg_len))) return HB_ERR_ARG;
    std::lock_guard<std::mutex> lk(w->mu);
    size_t off = 0;
    for (uint32_t k = 0; k < n_segs; k++) {
        fputc('>', w->f);
        fputs(id, w->f);
        if (n_segs == 1) fputc(' ', w->f); else fprintf(w->f, ":%u ", k);
        if (description) fputs(description, w->f);
        fputc('\n', w->f);
        fwrite(seqs + off, 1, seg_len[k], w->f);
        fputc('\n', w->f);
        off += seg_len[k];
        w->records++;
        w->bases += seg_len[k];
    }
    return HB_OK;
}
int hbh_fasta_close(hbh_fasta* w, uint64_t* records, uint64_t* bases) {
    if (!w) return HB_ERR_ARG;
    const int rc = fclose(w->f) == 0 ? HB_OK : HB_ERR_ARG;
    if (records) *records = w->records;
    if (bases) *bases = w->bases;
    delete w;
    return rc;
}

// ================================================================================================ the whole pipeline
// Bytes of the packed read store (2-bit words and one quality byte per base), which `host_store_above` is compared with
uint64_t hbh_reads_store_bytes(const hbh_reads* r) { return r->woff.back() * 8 + r->qoff.back(); }

// `herro inference --read-alns <alns_dir> -m <model> -b <batch> -t <threads> -d <devices> [-c cluster] <reads> <output>` over the C ABI.
// devices: n_dev CUDA device ids (targets are dealt to the devices' feature threads from one shared counter, like the
// reference's per-device worker groups pulling one channel, src/lib.rs:154-187).
// host_store_above: when the packed store is larger than this many bytes, the reads stay in host memory (one hb_read_store that every
// device attaches; the harness's own packed copy is freed once it exists), else every device gets an uploaded copy.
// times8: FASTQ load, pack, alignment ingest (wall), read-store upload or host-store creation + attach (max over devices),
// correction (first submit -> last result), FASTA close, total wall, corrected bases.
int hbh_inference(const char* reads_path, const char* alns_dir, const char* model, const char* output, uint32_t window, uint32_t batch,
                  int threads, const int* devices, int n_dev, const char* const* core, uint32_t n_core, const char* const* neighbour,
                  uint32_t n_neigh, int io_threads, uint64_t host_store_above, double* times8, uint64_t* counts4) {
    if (!reads_path || !alns_dir || !model || !output || !devices || n_dev < 1) return HB_ERR_ARG;
    const double t_begin = now_s();
    hbh_reads* R = nullptr;
    int rc = hbh_reads_load(reads_path, window, core, n_core, neighbour, n_neigh, io_threads, &R);
    if (rc) return rc;
    // Context creation (CUDA initialisation, weights) and the read-store upload of every device run while the alignment batches are
    // decompressed and parsed on the host: the two need nothing from each other (both only read `R`; the alignments need only
    // the names and lengths, so the packed words and qualities may go once a host store holds them).
    std::vector<hb_ctx*> ctx((size_t)n_dev, nullptr);
    hb_options opt{};
    opt.struct_size = sizeof opt; opt.window_size = window; opt.batch_size = batch;
    std::vector<double> t_up((size_t)n_dev, 0);
    hbh_alns* A = nullptr;
    hb_read_store* store = nullptr;
    auto cleanup = [&]() {
        for (hb_ctx* c : ctx) if (c) hb_destroy(c);
        if (store) hb_read_store_destroy(store);
        if (A) hbh_alns_free(A);
        hbh_reads_free(R);
    };
    std::atomic<int> bad{0};
    const bool host_store = hbh_reads_store_bytes(R) > host_store_above;
    double t_store = 0;
    std::string store_err;
    std::thread store_th;
    if (host_store)
        store_th = std::thread([&]() {
            const double t0 = now_s();
            if (hb_read_store_create(&store, hbh_reads_count(R), hbh_reads_word_ptrs(R), hbh_reads_lens(R), hbh_reads_qual_ptrs(R)) != HB_OK) {
                store_err = hb_last_error(nullptr);
                bad = HB_ERR_CUDA;
                return;
            }
            std::vector<uint64_t>().swap(R->words);
            std::vector<uint8_t>().swap(R->qual);
            R->word_ptr.assign(R->word_ptr.size(), nullptr);
            R->qual_ptr.assign(R->qual_ptr.size(), nullptr);
            t_store = now_s() - t0;
        });
    std::vector<std::thread> dev_th;
    for (int d = 0; d < n_dev; d++)
        dev_th.emplace_back([&, d]() {
            if (hb_create(&ctx[d], devices[d], model, &opt) != HB_OK) { bad = HB_ERR_CUDA; return; }
            if (host_store) return;
            const double t0 = now_s();
            if (hb_upload_reads(ctx[d], hbh_reads_count(R), hbh_reads_word_ptrs(R), hbh_reads_lens(R), hbh_reads_qual_ptrs(R)) != HB_OK) bad = HB_ERR_CUDA;
            t_up[d] = now_s() - t0;
        });
    const double t_al0 = now_s();
    rc = hbh_alns_load(alns_dir, R, core, n_core, io_threads, &A);
    const double t_ingest = now_s() - t_al0;
    const std::string ingest_err = rc ? t_err : std::string();
    for (auto& t : dev_th) t.join();
    if (host_store) {
        store_th.join();
        for (int d = 0; d < n_dev && !bad.load(); d++) {
            const double t0 = now_s();
            if (hb_attach_read_store(ctx[d], store) != HB_OK) bad = HB_ERR_CUDA;
            t_up[d] = t_store + now_s() - t0;
        }
    }
    if (rc) { t_err = ingest_err; cleanup(); return rc; }
    if (bad.load()) {
        t_err = "context creation / read-store upload failed";
        if (!store_err.empty()) t_err += ": " + store_err;
        for (hb_ctx* c : ctx) if (c) { t_err += std::string(": ") + hb_last_error(c); break; }
        if (const char* ce = hb_last_error(nullptr)) if (*ce) t_err += std::string(": ") + ce;
        cleanup();
        return bad.load();
    }
    hbh_fasta* W = nullptr;
    rc = hbh_fasta_open(output, &W);
    if (rc) { cleanup(); return rc; }
    const uint32_t n_tgt = hbh_alns_targets(A);
    std::atomic<uint32_t> next{0};
    std::atomic<int> fail{0};
    std::atomic<uint64_t> failed_targets{0}, answered{0};
    const double t_c0 = now_s();
    std::vector<std::thread> th;
    std::vector<std::atomic<int>> producers((size_t)n_dev);
    for (int d = 0; d < n_dev; d++) producers[d] = std::max(1, threads);
    for (int d = 0; d < n_dev; d++) {
        for (int t = 0; t < std::max(1, threads); t++)
            th.emplace_back([&, d]() {
                hb_bind_calling_thread(ctx[d]);
                for (;;) {
                    const uint32_t k = next.fetch_add(1);
                    if (k >= n_tgt || fail.load()) break;
                    const uint64_t a0 = A->tgt_off[k], a1 = A->tgt_off[k + 1];
                    const int r = hb_submit_alignments(ctx[d], A->tgt_rid[k], A->ovl.data() + a0, (uint32_t)(a1 - a0));
                    if (r == HB_ERR_INPUT) failed_targets.fetch_add(1);   // coordinates the reference would panic on: skip this read
                    else if (r != HB_OK) fail = r;
                }
                producers[d].fetch_sub(1);
            });
        th.emplace_back([&, d]() {  // consumer of device d
            hb_bind_calling_thread(ctx[d]);
            bool flushed = false;
            for (;;) {
                uint32_t rid = 0, n = 0;
                uint8_t* seqs = nullptr;
                uint32_t* lens = nullptr;
                const int r = hb_poll_corrected(ctx[d], &rid, &seqs, &lens, &n);
                if (r == 1) {
                    answered.fetch_add(1);
                    if (n) hbh_fasta_write(W, R->name_ptr[rid], hbh_reads_description(R, rid), seqs, lens, n);
                    hb_release_result(ctx[d], seqs);
                } else if (r == 0) {
                    if (producers[d].load() == 0) {
                        if (flushed) break;
                        const int f = hb_flush(ctx[d]);
                        if (f != HB_OK && f != HB_ERR_INPUT && f != HB_ERR_CAPACITY) fail = f;
                        flushed = true;
                    } else {
                        std::this_thread::sleep_for(std::chrono::microseconds(200));
                    }
                } else if (r == HB_ERR_INPUT || r == HB_ERR_CAPACITY) {
                    failed_targets.fetch_add(1);
                    fprintf(stderr, "herro_b200: skipped read %s: %s\n", rid < R->id.size() ? R->name_ptr[rid] : "?", hb_last_error(ctx[d]));
                } else {
                    fail = r;
                    if (flushed) break;
                }
            }
        });
    }
    for (auto& t : th) t.join();
    const double t_correct = now_s() - t_c0;
    const double t_w0 = now_s();
    uint64_t records = 0, bases = 0;
    hbh_fasta_close(W, &records, &bases);
    const double t_close = now_s() - t_w0;
    if (times8) {
        times8[0] = R->t_load; times8[1] = R->t_pack; times8[2] = t_ingest; times8[3] = *std::max_element(t_up.begin(), t_up.end());
        times8[4] = t_correct; times8[5] = t_close; times8[6] = now_s() - t_begin; times8[7] = (double)bases;
    }
    if (counts4) { counts4[0] = hbh_reads_count(R); counts4[1] = n_tgt; counts4[2] = records; counts4[3] = failed_targets.load(); }
    rc = fail.load();
    if (rc) t_err = std::string("correction failed: ") + hb_last_error(ctx[0]);
    cleanup();
    return rc;
}

}  // extern "C"
