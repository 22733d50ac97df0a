// io.cpp — the host data plane around the hot path, natively and multi-threaded (SURVEY.md §8f-2, §8f-4):
//
//   hbh_reads_*    FASTQ (plain or .gz) -> read ids, descriptions, qualities, 2-bit packed sequences in the HAECSeq layout
//                  (haec_io::get_reads, src/haec_io.rs:37-75,121-136): reads shorter than the window are dropped (:48), the
//                  id is split from the description at the first space / tab (:52-54), cluster filter (:64-70)
//   hbh_alns_*     a `--read-alns` directory of *.oec.zst batches -> alignments grouped by target
//                  (overlaps::read_batches + parse_paf, src/overlaps.rs:288-323,117-202): header lines skipped, unknown read
//                  names skipped, core filter on the target, self overlaps dropped, only the first line of an ordered
//                  (query, target) pair per batch file kept.  The reference decodes and parses batch files one after the
//                  other on one thread; here workers decompress (libzstd through dlopen: the image ships the library but no
//                  header) and parse upcoming files while earlier ones are used (hbh_alns_stream_*), within a budget of host
//                  memory; hbh_alns_load is the same stream with no budget, merged.
//   hbh_paf_*      an overlap-only PAF (plain or .gz, minimap2 without -c), read in chunks of lines under parse_paf's admission
//                  rules: unknown read names and self overlaps skipped, any cg:Z: ignored, repeated pairs kept
//   hbh_batches_*  the write mode of generate_batches (src/overlaps.rs:264-285, scripts/batch.py): <k>.oec.zst holds the k-th run of
//                  batch_size loaded reads (header: the count, then one id per line) and every line whose target is among them
//   hbh_align      `herro align`: hbh_paf_* -> hb_align_overlaps -> hbh_batches_*
//   hbh_fasta_*    correction_writer / write_sequence (src/lib.rs:267-317): `>id[:k] description\n seq\n`
//   hbh_inference  the whole `herro inference --read-alns` pipeline over the public C ABI of libherro_b200: FASTQ ingest ->
//                  hb_upload_reads (or one host read store for all devices) -> feature threads (hb_submit_alignments) fed by the
//                  alignment stream -> consumer (hb_poll_corrected) -> FASTA, with the time of every stage reported.
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
#include <condition_variable>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <deque>
#include <memory>
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
    void* (*createCCtx)() = nullptr;
    size_t (*freeCCtx)(void*) = nullptr;
    size_t (*compressStream2)(void*, ZOutBuf*, ZInBuf*, int) = nullptr;  // ZSTD_e_continue 0, ZSTD_e_end 2
    bool ok = false;
    bool ok_c = false;
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
        r.createCCtx = (void* (*)())dlsym(r.h, "ZSTD_createCCtx");
        r.freeCCtx = (size_t(*)(void*))dlsym(r.h, "ZSTD_freeCCtx");
        r.compressStream2 = (size_t(*)(void*, ZOutBuf*, ZInBuf*, int))dlsym(r.h, "ZSTD_compressStream2");
        r.ok = r.createDStream && r.freeDStream && r.initDStream && r.decompressStream && r.isError;
        r.ok_c = r.createCCtx && r.freeCCtx && r.compressStream2 && r.isError;
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
        if (in.pos == in.size && (r == 0 || ob.pos < ob.size)) break;  // input consumed, and the last frame ended or the output
                                                                      // buffer was not the limit
    }
    z.freeDStream(ds);
    out.resize(produced);
    // a buffer that grew past the text is trimmed: the stream's budget counts the bytes a file holds
    if (out.capacity() > produced + produced / 16) out.shrink_to_fit();
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

struct AlnStream;
struct hbh_alns_stream;

struct hbh_alns {
    std::vector<std::vector<uint8_t>> text;  // decompressed batch files (the CIGARs point into them)
    std::vector<hb_overlap> ovl;             // grouped by target
    std::vector<uint32_t> tgt_rid;
    std::vector<uint64_t> tgt_off;           // [n_targets+1] into ovl
    double t_decode = 0, t_parse = 0;
    uint64_t lines = 0, kept = 0, compressed_bytes = 0, text_bytes = 0;
    uint32_t files = 0;
    std::string source;                      // the batch file of a streamed file; empty for a merged load
    std::shared_ptr<AlnStream> stream;       // the stream whose budget this file holds (NULL for a merged load)
    uint64_t budget_bytes = 0;               // this file's share of that budget
};

struct hbh_fasta {
    FILE* f = nullptr;
    std::mutex mu;
    uint64_t records = 0, bases = 0;
};

extern "C" {

const char* hbh_last_error() { return t_err.c_str(); }
void hbh_alns_free(hbh_alns* a);

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

// Group a file's overlaps by target, in order of first appearance (the reference's HashMap order is arbitrary, F8), appended to A.
void group_by_target(const std::vector<hb_overlap>& ovl, hbh_alns& A) {
    std::unordered_map<uint32_t, uint32_t> slot;
    std::vector<uint32_t> cnt;
    std::vector<uint32_t> tids;
    for (const hb_overlap& o : ovl) {
        auto it = slot.find(o.tid);
        if (it == slot.end()) { slot.emplace(o.tid, (uint32_t)cnt.size()); cnt.push_back(1); tids.push_back(o.tid); }
        else cnt[it->second]++;
    }
    if (A.tgt_off.empty()) A.tgt_off.push_back(0);
    const size_t base = A.ovl.size();
    std::vector<uint64_t> start(cnt.size() + 1, 0);
    for (size_t k = 0; k < cnt.size(); k++) start[k + 1] = start[k] + cnt[k];
    A.ovl.resize(base + ovl.size());
    std::vector<uint64_t> fill(start.begin(), start.end() - 1);
    for (const hb_overlap& o : ovl) A.ovl[base + fill[slot[o.tid]]++] = o;
    for (size_t k = 0; k < cnt.size(); k++) {
        A.tgt_rid.push_back(tids[k]);
        A.tgt_off.push_back(base + start[k + 1]);
    }
}

bool list_batches(const char* dir, std::vector<std::string>& files) {
    DIR* d = opendir(dir);
    if (!d) { t_err = std::string("cannot open directory ") + dir; return false; }
    while (dirent* e = readdir(d)) {
        const std::string nme = e->d_name;
        if (nme.size() > 8 && nme.compare(nme.size() - 8, 8, ".oec.zst") == 0) files.push_back(std::string(dir) + "/" + nme);
    }
    closedir(d);
    std::sort(files.begin(), files.end());
    return true;
}

uint64_t physical_memory() { return (uint64_t)sysconf(_SC_PHYS_PAGES) * (uint64_t)sysconf(_SC_PAGE_SIZE); }

// The text a batch file will decompress to: the size its first zstd frame records, else four times the file (a guess; the
// reservation is corrected once the file is decoded).
uint64_t text_estimate(const std::string& path) {
    struct stat st;
    if (stat(path.c_str(), &st) != 0) return 0;
    uint8_t head[18];
    const int fd = open(path.c_str(), O_RDONLY);
    if (fd < 0) return 0;
    const ssize_t n = pread(fd, head, sizeof head, 0);
    close(fd);
    const Zstd& z = zstd();
    if (n > 0 && z.getFrameContentSize) {
        const unsigned long long cs = z.getFrameContentSize(head, (size_t)n);
        if (cs != 0ull - 1 && cs != 0ull - 2) return (uint64_t)cs;
    }
    return (uint64_t)st.st_size * 4;
}
}  // namespace

// The streaming reader.  Workers take the batch files in sorted name order; a worker starts the next file only while the bytes in
// flight (decompressed text plus grouped hb_overlap arrays of every file started and not yet freed) are below the budget, or when no
// file is in flight at all, so one file larger than the budget still runs.  A file decoded early waits in its slot until every
// earlier file has been handed out.  Starting a file reserves the text it is expected to decompress to (text_estimate), so workers
// decoding side by side cannot all start at once under the budget; the charge becomes the file's text once decoded, then its text
// plus its overlap array, and hbh_alns_free releases it.  That may happen after the stream is closed: every streamed hbh_alns keeps
// the shared state alive.
struct AlnStream {
    const hbh_reads* R = nullptr;
    std::vector<std::string> core_names;          // owned copies: the workers outlive hbh_alns_stream_open's arguments
    std::unordered_set<std::string_view> core_set;
    bool use_core = false;
    std::vector<std::string> files;
    std::vector<uint64_t> estimate;               // text bytes a file is expected to hold, reserved when a worker starts it
    uint64_t budget = 0;
    std::mutex mu;
    std::condition_variable cv;
    struct Slot { hbh_alns* a = nullptr; bool done = false; std::string err; };
    std::vector<Slot> slot;
    size_t next_start = 0, next_out = 0, error_at = SIZE_MAX;
    uint64_t in_flight = 0, peak = 0;
    uint32_t files_in_flight = 0, peak_files = 0, parsed = 0;
    double t_open = 0, t_last_parsed = 0;
    bool stop = false;
    std::vector<std::thread> workers;

    void charge(hbh_alns& A, uint64_t bytes) {  // A now holds `bytes` (until now it held A.budget_bytes)
        std::lock_guard<std::mutex> lk(mu);
        in_flight = in_flight - A.budget_bytes + bytes;
        A.budget_bytes = bytes;
        peak = std::max(peak, in_flight);
    }
    void release(const hbh_alns& A) {  // under mu
        in_flight -= A.budget_bytes;
        files_in_flight--;
        cv.notify_all();
    }
    static void work(const std::shared_ptr<AlnStream>& sp) {
        AlnStream& S = *sp;
        for (;;) {
            size_t i;
            {
                std::unique_lock<std::mutex> lk(S.mu);
                S.cv.wait(lk, [&] { return S.stop || S.next_start >= S.files.size() || S.next_start > S.error_at ||
                                           S.files_in_flight == 0 || S.in_flight < S.budget; });
                if (S.stop || S.next_start >= S.files.size() || S.next_start > S.error_at) return;
                i = S.next_start++;
                S.files_in_flight++;
                S.peak_files = std::max(S.peak_files, S.files_in_flight);
                // the reservation keeps the other workers from starting files past the budget while this one decodes
                S.in_flight += S.estimate[i];
                S.peak = std::max(S.peak, S.in_flight);
            }
            auto* A = new hbh_alns();
            A->budget_bytes = S.estimate[i];
            A->files = 1;
            A->source = S.files[i];
            A->stream = sp;
            std::string err;
            bool ok = false;
            {
                const double t0 = now_s();
                FileBytes fb;
                A->text.emplace_back();
                if (!load_file(S.files[i], fb)) {
                    err = t_err;
                } else {
                    A->compressed_bytes = fb.n;
                    ok = zstd_decompress(fb.p, fb.n, A->text.back());
                    if (!ok) err = t_err + " in " + S.files[i];
                }
                A->t_decode = now_s() - t0;
            }
            if (ok) {
                A->text_bytes = A->text.back().size();
                S.charge(*A, A->text_bytes);
                const double t1 = now_s();
                FileAlns fa;
                parse_batch(S.R, S.use_core ? &S.core_set : nullptr, A->text.back(), fa);
                if (fa.ok) {
                    A->lines = fa.lines;
                    A->kept = fa.ovl.size();
                    group_by_target(fa.ovl, *A);
                    S.charge(*A, A->text_bytes + A->ovl.size() * sizeof(hb_overlap));
                } else {
                    ok = false;
                    err = fa.err + " in " + S.files[i];
                }
                A->t_parse = now_s() - t1;
            }
            std::unique_lock<std::mutex> lk(S.mu);
            Slot& sl = S.slot[i];
            sl.done = true;
            S.parsed++;
            S.t_last_parsed = now_s();
            if (ok) {
                sl.a = A;
                S.cv.notify_all();
            } else {
                sl.err = err;
                S.error_at = std::min(S.error_at, i);
                S.release(*A);
                A->stream.reset();
                lk.unlock();
                delete A;
            }
        }
    }
};

struct hbh_alns_stream { std::shared_ptr<AlnStream> s; };

// Bytes the streaming reader may hold when the caller passes a budget of 0: 1/8 of physical memory.
uint64_t hbh_alns_default_budget() { return std::max<uint64_t>(physical_memory() / 8, 1); }

// Starts up to `threads` workers that decompress and parse the *.oec.zst files of `dir` ahead of the caller, within `budget_bytes`
// (0: hbh_alns_default_budget()).  core / n_core as hbh_alns_load.  The caller frees every file hbh_alns_stream_next hands out with
// hbh_alns_free: files held past the budget stop the workers, so a caller that keeps them all must pass a budget that covers them.
int hbh_alns_stream_open(const char* dir, const hbh_reads* reads, const char* const* core, uint32_t n_core, int threads,
                         uint64_t budget_bytes, hbh_alns_stream** out) {
    if (!dir || !reads || !out) return HB_ERR_ARG;
    *out = nullptr;
    auto sp = std::make_shared<AlnStream>();
    AlnStream& S = *sp;
    if (!list_batches(dir, S.files)) return HB_ERR_ARG;
    S.R = reads;
    if (core) {
        S.use_core = true;
        S.core_names.assign(core, core + n_core);
        for (const std::string& c : S.core_names) S.core_set.insert(c);
    }
    S.budget = budget_bytes ? budget_bytes : hbh_alns_default_budget();
    S.slot.resize(S.files.size());
    for (const std::string& f : S.files) S.estimate.push_back(text_estimate(f));
    S.t_open = now_s();
    S.t_last_parsed = S.t_open;
    const int n_workers = std::max(1, std::min<int>(threads, (int)S.files.size()));
    for (int i = 0; i < n_workers && !S.files.empty(); i++) S.workers.emplace_back(AlnStream::work, sp);
    *out = new hbh_alns_stream{sp};
    return HB_OK;
}

// The next file's alignments, in sorted name order: *a is an ordinary hbh_alns (the hbh_alns_* accessors apply), or NULL after the
// last file.  A file that cannot be read, decompressed or parsed returns HB_ERR_INPUT naming it, here and on every later call.
int hbh_alns_stream_next(hbh_alns_stream* s, hbh_alns** a) {
    if (!s || !a) return HB_ERR_ARG;
    *a = nullptr;
    AlnStream& S = *s->s;
    std::unique_lock<std::mutex> lk(S.mu);
    if (S.next_out >= S.files.size()) return HB_OK;
    S.cv.wait(lk, [&] { return S.slot[S.next_out].done; });
    AlnStream::Slot& sl = S.slot[S.next_out];
    if (!sl.a) { t_err = sl.err; return HB_ERR_INPUT; }
    *a = sl.a;
    sl.a = nullptr;
    S.next_out++;
    return HB_OK;
}

// Stops the workers and frees the files not handed out.  Files already handed out stay valid until their hbh_alns_free.
void hbh_alns_stream_close(hbh_alns_stream* s) {
    if (!s) return;
    AlnStream& S = *s->s;
    {
        std::lock_guard<std::mutex> lk(S.mu);
        S.stop = true;
        S.cv.notify_all();
    }
    for (auto& t : S.workers) t.join();
    std::vector<hbh_alns*> left;
    {
        std::lock_guard<std::mutex> lk(S.mu);
        for (auto& sl : S.slot) if (sl.a) { left.push_back(sl.a); sl.a = nullptr; }
    }
    for (hbh_alns* a : left) hbh_alns_free(a);
    delete s;
}

// counts6: peak bytes in flight, bytes in flight now, budget, files, files parsed (or failed), peak files in flight.
// ingest_s: seconds from hbh_alns_stream_open to the last file parsed so far.
void hbh_alns_stream_stats(hbh_alns_stream* s, uint64_t* counts6, double* ingest_s) {
    AlnStream& S = *s->s;
    std::lock_guard<std::mutex> lk(S.mu);
    if (counts6) {
        counts6[0] = S.peak; counts6[1] = S.in_flight; counts6[2] = S.budget; counts6[3] = S.files.size(); counts6[4] = S.parsed;
        counts6[5] = S.peak_files;
    }
    if (ingest_s) *ingest_s = S.t_last_parsed - S.t_open;
}

// Every file of `dir` merged into one hbh_alns: the stream with no budget, its files concatenated in order.  A target named in
// several files is sent once per file, like the reference's per-batch maps.
int hbh_alns_load(const char* dir, const hbh_reads* reads, const char* const* core, uint32_t n_core, int threads, hbh_alns** out) {
    if (!dir || !reads || !out) return HB_ERR_ARG;
    *out = nullptr;
    hbh_alns_stream* s = nullptr;
    int rc = hbh_alns_stream_open(dir, reads, core, n_core, threads, UINT64_MAX, &s);
    if (rc) return rc;
    auto* A = new hbh_alns();
    A->tgt_off.push_back(0);
    for (;;) {
        hbh_alns* f = nullptr;
        rc = hbh_alns_stream_next(s, &f);
        if (rc) { hbh_alns_stream_close(s); delete A; return rc; }
        if (!f) break;
        const uint64_t base = A->ovl.size();
        A->ovl.insert(A->ovl.end(), f->ovl.begin(), f->ovl.end());
        A->tgt_rid.insert(A->tgt_rid.end(), f->tgt_rid.begin(), f->tgt_rid.end());
        for (size_t k = 1; k < f->tgt_off.size(); k++) A->tgt_off.push_back(base + f->tgt_off[k]);
        for (auto& t : f->text) A->text.push_back(std::move(t));  // the buffers move, so the CIGAR pointers stay valid
        A->t_decode += f->t_decode; A->t_parse += f->t_parse; A->lines += f->lines; A->kept += f->kept;
        A->compressed_bytes += f->compressed_bytes; A->text_bytes += f->text_bytes;
        A->files++;
        hbh_alns_free(f);
    }
    hbh_alns_stream_close(s);
    *out = A;
    return HB_OK;
}

void hbh_alns_free(hbh_alns* a) {
    if (!a) return;
    if (a->stream) {
        std::lock_guard<std::mutex> lk(a->stream->mu);
        a->stream->release(*a);
    }
    delete a;
}
uint32_t hbh_alns_targets(const hbh_alns* a) { return (uint32_t)a->tgt_rid.size(); }
const uint32_t* hbh_alns_target_rids(const hbh_alns* a) { return a->tgt_rid.data(); }
const uint64_t* hbh_alns_target_offsets(const hbh_alns* a) { return a->tgt_off.data(); }
const hb_overlap* hbh_alns_overlaps(const hbh_alns* a) { return a->ovl.data(); }
// The batch file a streamed hbh_alns came from; "" for hbh_alns_load's merged result.
const char* hbh_alns_source(const hbh_alns* a) { return a->source.c_str(); }
// stats6: sum of per-file decode seconds, sum of per-file parse seconds, PAF lines, alignments kept, compressed bytes, text bytes
void hbh_alns_stats(const hbh_alns* a, double* stats6) {
    stats6[0] = a->t_decode; stats6[1] = a->t_parse; stats6[2] = (double)a->lines; stats6[3] = (double)a->kept;
    stats6[4] = (double)a->compressed_bytes; stats6[5] = (double)a->text_bytes;
}
// The bytes a streamed file holds of its stream's budget: its text plus its grouped hb_overlap array.
uint64_t hbh_alns_budget_bytes(const hbh_alns* a) { return a->budget_bytes; }

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
// devices: n_dev CUDA device ids.  The feature threads of every device pull targets from one shared queue that the streaming reader
// (hbh_alns_stream_*) fills file by file, like the reference's per-device worker groups pulling one channel that alignment_reader
// fills a batch file at a time (src/lib.rs:154-187, src/overlaps.rs:325-375).  Correction starts once the contexts exist and the
// first file is parsed, while later files are still being decoded; the feature thread whose hb_submit_alignments returns for a
// file's last target frees the file (hb_submit_alignments copies the CIGAR bytes), which returns its bytes to the reader's budget.
// host_store_above: when the packed store is larger than this many bytes, the reads stay in host memory (one hb_read_store that every
// device attaches; the harness's own packed copy is freed once it exists), else every device gets an uploaded copy.
// aln_budget: bytes of decompressed text and hb_overlap arrays the reader may hold at once (0: hbh_alns_default_budget(), 1/8 of
// physical memory); one file larger than the budget is still read whole.
// An ingest error (a file that cannot be read or decompressed, a bad header, a malformed line) ends the hand-out of targets at that
// file: the targets of the files before it are submitted, flushed and their records written, then the call returns HB_ERR_INPUT
// naming the file.  The output file then holds the records of the targets before the error (the reference panics at that point).
// times9: FASTQ load, pack, alignment ingest (wall, first file opened -> last file parsed), read-store upload or host-store creation +
// attach (max over devices), correction (feature threads started -> last result), FASTA close, total wall, corrected bases, first submit
// (seconds from the start of the call to the first hb_submit_alignments, -1 when there was none).
// counts6: reads, targets, records, failed targets, peak bytes the alignment reader held, its budget.
int hbh_inference(const char* reads_path, const char* alns_dir, const char* model, const char* output, uint32_t window, uint32_t batch,
                  int threads, const int* devices, int n_dev, const char* const* core, uint32_t n_core, const char* const* neighbour,
                  uint32_t n_neigh, int io_threads, uint64_t host_store_above, uint64_t aln_budget, double* times9, uint64_t* counts6) {
    if (!reads_path || !alns_dir || !model || !output || !devices || n_dev < 1) return HB_ERR_ARG;
    const double t_begin = now_s();
    hbh_reads* R = nullptr;
    int rc = hbh_reads_load(reads_path, window, core, n_core, neighbour, n_neigh, io_threads, &R);
    if (rc) return rc;
    // Context creation (CUDA initialisation, weights) and the read-store upload of every device run while the first alignment batches
    // are decompressed and parsed on the host: the two need nothing from each other (both only read `R`; the alignments need only
    // the names and lengths, so the packed words and qualities may go once a host store holds them).
    std::vector<hb_ctx*> ctx((size_t)n_dev, nullptr);
    hb_options opt{};
    opt.struct_size = sizeof opt; opt.window_size = window; opt.batch_size = batch;
    std::vector<double> t_up((size_t)n_dev, 0);
    hbh_alns_stream* S = nullptr;
    hb_read_store* store = nullptr;
    auto cleanup = [&]() {
        if (S) hbh_alns_stream_close(S);
        for (hb_ctx* c : ctx) if (c) hb_destroy(c);
        if (store) hb_read_store_destroy(store);
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
    rc = hbh_alns_stream_open(alns_dir, R, core, n_core, io_threads, aln_budget, &S);
    const std::string open_err = rc ? t_err : std::string();
    for (auto& t : dev_th) t.join();
    if (host_store) {
        store_th.join();
        for (int d = 0; d < n_dev && !bad.load(); d++) {
            const double t0 = now_s();
            if (hb_attach_read_store(ctx[d], store) != HB_OK) bad = HB_ERR_CUDA;
            t_up[d] = t_store + now_s() - t0;
        }
    }
    if (rc) { t_err = open_err; cleanup(); return rc; }
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
    // The shared queue: parsed files in order, each handing out its targets one at a time.  `left` counts the targets of a file not
    // yet returned from hb_submit_alignments (or abandoned); whoever takes it to zero frees the file.
    struct QFile {
        hbh_alns* a;
        uint32_t n, next;
        std::atomic<uint32_t> left;
        QFile(hbh_alns* a_, uint32_t n_) : a(a_), n(n_), next(0), left(n_) {}
    };
    std::mutex qmu;
    std::condition_variable qcv;
    std::deque<QFile*> queue;
    bool feed_done = false, abandoned = false;
    auto done = [](QFile* f, uint32_t k) {
        if (f->left.fetch_sub(k) == k) { hbh_alns_free(f->a); delete f; }
    };
    auto abandon = [&]() {  // under qmu: no further targets are handed out, and the queued files go back to the budget
        abandoned = true;
        for (QFile* f : queue) { const uint32_t k = f->n - f->next; f->next = f->n; done(f, k); }
        queue.clear();
        qcv.notify_all();
    };
    uint64_t n_tgt = 0;
    std::atomic<int> fail{0};
    std::atomic<bool> submitted{false};
    double t_first_submit = -1;
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
                    QFile* f;
                    uint32_t k;
                    {
                        std::unique_lock<std::mutex> lk(qmu);
                        // the timeout only bounds how late a failure set by another thread is noticed
                        qcv.wait_for(lk, std::chrono::milliseconds(20), [&] { return !queue.empty() || feed_done || abandoned || fail.load(); });
                        if (fail.load() && !abandoned) abandon();
                        if (abandoned || (queue.empty() && feed_done)) break;
                        if (queue.empty()) continue;
                        f = queue.front();
                        k = f->next++;
                        if (f->next == f->n) queue.pop_front();
                    }
                    if (!submitted.exchange(true)) t_first_submit = now_s() - t_begin;
                    const hbh_alns* A = f->a;
                    const uint64_t a0 = A->tgt_off[k], a1 = A->tgt_off[k + 1];
                    const int r = hb_submit_alignments(ctx[d], A->tgt_rid[k], A->ovl.data() + a0, (uint32_t)(a1 - a0));
                    done(f, 1);
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
    // This thread feeds the queue from the stream: it blocks while the next file is decoded or the budget is held.
    int ingest_rc = 0;
    std::string ingest_err;
    while (!fail.load()) {
        hbh_alns* a = nullptr;
        const int r = hbh_alns_stream_next(S, &a);
        if (r) { ingest_rc = r; ingest_err = t_err; break; }
        if (!a) break;
        const uint32_t n = hbh_alns_targets(a);
        n_tgt += n;
        if (n == 0) { hbh_alns_free(a); continue; }
        std::lock_guard<std::mutex> lk(qmu);
        if (abandoned) { hbh_alns_free(a); break; }
        queue.push_back(new QFile(a, n));
        qcv.notify_all();
    }
    {
        std::lock_guard<std::mutex> lk(qmu);
        feed_done = true;  // after an ingest error the files before the broken one are still corrected: the hand-out ends there
        qcv.notify_all();
    }
    uint64_t st[6] = {0, 0, 0, 0, 0, 0};
    double t_ingest = 0;
    hbh_alns_stream_stats(S, st, &t_ingest);
    hbh_alns_stream_close(S);
    S = nullptr;
    for (auto& t : th) t.join();
    {
        std::lock_guard<std::mutex> lk(qmu);
        abandon();  // nothing is left unless every feature thread stopped on a failure
    }
    const double t_correct = now_s() - t_c0;
    const double t_w0 = now_s();
    uint64_t records = 0, bases = 0;
    hbh_fasta_close(W, &records, &bases);
    const double t_close = now_s() - t_w0;
    if (times9) {
        times9[0] = R->t_load; times9[1] = R->t_pack; times9[2] = t_ingest; times9[3] = *std::max_element(t_up.begin(), t_up.end());
        times9[4] = t_correct; times9[5] = t_close; times9[6] = now_s() - t_begin; times9[7] = (double)bases;
        times9[8] = t_first_submit;
    }
    if (counts6) {
        counts6[0] = hbh_reads_count(R); counts6[1] = n_tgt; counts6[2] = records; counts6[3] = failed_targets.load();
        counts6[4] = st[0]; counts6[5] = st[2];
    }
    rc = fail.load();
    if (rc) t_err = std::string("correction failed: ") + hb_last_error(ctx[0]);
    else if (ingest_rc) { rc = ingest_rc; t_err = ingest_err; }
    cleanup();
    return rc;
}

}  // extern "C"

// ================================================================================================ overlap-only PAF -> aligned batches
struct hbh_paf {
    gzFile g = nullptr;               // gzopen reads plain files as they are
    std::vector<uint8_t> buf;         // the current chunk's lines (the admitted lines' mapq fields lie in it)
    size_t carry = 0;                 // bytes of an unfinished line kept from the previous read
    bool eof = false;
    const hbh_reads* R = nullptr;
    std::vector<hb_overlap> ovl;      // the admitted lines of the current chunk, cigar NULL
    std::vector<std::pair<uint32_t, uint32_t>> mapq;  // column 12 of each admitted line: offset into buf, length
    uint64_t lines = 0, skipped = 0, bytes = 0;
};

struct hbh_batches {
    struct File { FILE* f = nullptr; void* cctx = nullptr; std::string pending; uint64_t lines = 0; };
    std::vector<File> files;
    const hbh_reads* R = nullptr;
    uint32_t batch_size = 0;
    std::vector<uint8_t> zbuf;
    uint64_t written = 0;
};

namespace {

constexpr size_t PAF_READ = 16u << 20;

bool flush_batch(hbh_batches* B, hbh_batches::File& F, bool end) {
    const Zstd& z = zstd();
    ZInBuf in{F.pending.data(), F.pending.size(), 0};
    for (;;) {
        ZOutBuf out{B->zbuf.data(), B->zbuf.size(), 0};
        const size_t r = z.compressStream2(F.cctx, &out, &in, end ? 2 : 0);
        if (z.isError(r)) { t_err = "zstd compression failed"; return false; }
        if (out.pos && fwrite(B->zbuf.data(), 1, out.pos, F.f) != out.pos) { t_err = "write failed"; return false; }
        if (end ? r == 0 : in.pos == in.size) break;
    }
    F.pending.clear();
    return true;
}

}  // namespace

extern "C" {

int hbh_batches_close(hbh_batches* B, uint64_t* lines_per_batch);

// An overlap-only PAF (plain or gzip).  Lines are admitted as parse_paf admits them (src/overlaps.rs:117-202) with reads' names
// (reads shorter than the window are not loaded, so their lines go), self overlaps skipped; a cg:Z: field is ignored.
int hbh_paf_open(const char* path, const hbh_reads* reads, hbh_paf** out) {
    if (!path || !reads || !out) { t_err = "null pointer"; return HB_ERR_ARG; }
    gzFile g = gzopen(path, "rb");
    if (!g) { t_err = std::string("cannot open ") + path; return HB_ERR_INPUT; }
    gzbuffer(g, 1 << 20);
    hbh_paf* P = new hbh_paf;
    P->g = g;
    P->R = reads;
    *out = P;
    return HB_OK;
}

// The next chunk: up to max_lines admitted lines (fewer at the end of the file; 0 once it is read).  *n_out is their count; their
// overlaps (hbh_paf_overlaps) stay valid until the next call.
int hbh_paf_next(hbh_paf* P, uint32_t max_lines, uint32_t* n_out) {
    if (!P || !n_out || !max_lines) { t_err = "null pointer or zero max_lines"; return HB_ERR_ARG; }
    P->ovl.clear();
    P->mapq.clear();
    *n_out = 0;
    // keep reading until max_lines are admitted or the file ends; the unparsed tail of the buffer carries over
    std::vector<uint8_t>& b = P->buf;
    size_t pos = 0;
    if (P->carry) { memmove(b.data(), b.data() + b.size() - P->carry, P->carry); b.resize(P->carry); P->carry = 0; }
    else b.clear();
    while (P->ovl.size() < max_lines) {
        const uint8_t* base = b.data();
        const uint8_t* e = base + b.size();
        const uint8_t* p = base + pos;
        const uint8_t* nl = (const uint8_t*)memchr(p, '\n', (size_t)(e - p));
        if (!nl) {
            if (P->eof) {
                if (p == e) break;
                b.push_back('\n');  // a last line without a newline
                continue;
            }
            const size_t old = b.size();
            b.resize(old + PAF_READ);
            const int r = gzread(P->g, b.data() + old, (unsigned)PAF_READ);
            if (r < 0) { t_err = "PAF read error"; return HB_ERR_INPUT; }
            b.resize(old + (size_t)r);
            P->bytes += (uint64_t)r;
            if (r == 0) P->eof = true;
            continue;
        }
        pos = (size_t)(nl + 1 - base);
        const uint8_t* le = nl;
        if (le > p && le[-1] == '\r') le--;
        if (le == p) continue;
        P->lines++;
        const uint8_t* f[12][2];
        int nf = 0;
        for (const uint8_t* c = p; nf < 12;) {
            const uint8_t* t = (const uint8_t*)memchr(c, '\t', (size_t)(le - c));
            if (!t) t = le;
            f[nf][0] = c; f[nf][1] = t;
            nf++;
            if (t == le) break;
            c = t + 1;
        }
        if (nf < 12) { t_err = "PAF line " + std::to_string(P->lines) + ": fewer than 12 columns"; return HB_ERR_INPUT; }
        auto qit = P->R->name_to_id.find(std::string_view((const char*)f[0][0], (size_t)(f[0][1] - f[0][0])));
        auto tit = P->R->name_to_id.find(std::string_view((const char*)f[5][0], (size_t)(f[5][1] - f[5][0])));
        if (qit == P->R->name_to_id.end() || tit == P->R->name_to_id.end() || qit->second == tit->second) { P->skipped++; continue; }
        hb_overlap o{};
        o.qid = qit->second;
        o.tid = tit->second;
        const uint8_t sc = f[4][0] < f[4][1] ? *f[4][0] : 0;
        if (!parse_u32(f[1][0], f[1][1], o.qlen) || !parse_u32(f[2][0], f[2][1], o.qstart) || !parse_u32(f[3][0], f[3][1], o.qend) ||
            !parse_u32(f[6][0], f[6][1], o.tlen) || !parse_u32(f[7][0], f[7][1], o.tstart) || !parse_u32(f[8][0], f[8][1], o.tend) ||
            (sc != '+' && sc != '-')) {
            t_err = "PAF line " + std::to_string(P->lines) + ": malformed number or strand";
            return HB_ERR_INPUT;
        }
        o.strand = sc == '-';
        P->ovl.push_back(o);
        P->mapq.emplace_back((uint32_t)(f[11][0] - base), (uint32_t)(f[11][1] - f[11][0]));
    }
    // the unparsed rest carries over to the next call
    P->carry = b.size() - pos;
    *n_out = (uint32_t)P->ovl.size();
    return HB_OK;
}

const hb_overlap* hbh_paf_overlaps(const hbh_paf* P) { return P->ovl.data(); }
void hbh_paf_stats(const hbh_paf* P, uint64_t* counts3) { counts3[0] = P->lines; counts3[1] = P->skipped; counts3[2] = P->bytes; }
void hbh_paf_close(hbh_paf* P) {
    if (!P) return;
    if (P->g) gzclose(P->g);
    delete P;
}

// <dir>/<k>.oec.zst for k < ceil(reads / batch_size), each starting with its header
int hbh_batches_open(const char* dir, const hbh_reads* reads, uint32_t batch_size, hbh_batches** out) {
    if (!dir || !reads || !out || !batch_size) { t_err = "null pointer or zero batch size"; return HB_ERR_ARG; }
    if (!zstd().ok_c) { t_err = "libzstd with ZSTD_compressStream2 not found"; return HB_ERR_STATE; }
    mkdir(dir, 0777);
    hbh_batches* B = new hbh_batches;
    B->R = reads;
    B->batch_size = batch_size;
    B->zbuf.resize(1 << 17);
    const uint32_t n = (uint32_t)reads->id.size();
    for (uint32_t k = 0; (uint64_t)k * batch_size < n; k++) {
        hbh_batches::File F;
        const std::string path = std::string(dir) + "/" + std::to_string(k) + ".oec.zst";
        F.f = fopen(path.c_str(), "wb");
        F.cctx = zstd().createCCtx();
        const uint32_t r0 = k * batch_size, r1 = std::min<uint64_t>((uint64_t)r0 + batch_size, n);
        F.pending = std::to_string(r1 - r0) + "\n";
        for (uint32_t r = r0; r < r1; r++) { F.pending += reads->id[r]; F.pending += '\n'; }
        const bool ok = F.f && F.cctx;
        B->files.push_back(std::move(F));
        if (!ok) { t_err = "cannot create " + path; hbh_batches_close(B, nullptr); return HB_ERR_INPUT; }
    }
    *out = B;
    return HB_OK;
}

// Append the lines of one chunk: line i of `paf`'s current chunk with the coordinates and CIGAR of aligned[i] (hb_align_fetch's
// `out`), matches[i] as column 10 and the sum of the CIGAR's op lengths as column 11, to the batch of its target, in input order.
// Lines with status[i] < 0 are not written.
int hbh_batches_write(hbh_batches* B, const hbh_paf* paf, const hb_overlap* aligned, const int32_t* status, const uint32_t* matches,
                      uint32_t n) {
    if (!B || !paf || (n && (!aligned || !status || !matches)) || n > paf->ovl.size()) { t_err = "bad arguments"; return HB_ERR_ARG; }
    const hbh_reads* R = B->R;
    for (uint32_t i = 0; i < n; i++) {
        if (status[i] < 0) continue;
        const hb_overlap& o = aligned[i];
        uint64_t block = 0, v = 0;
        for (uint32_t c = 0; c < o.cigar_len; c++) {
            const uint8_t ch = o.cigar[c];
            if (ch >= '0' && ch <= '9') v = v * 10 + (ch - '0');
            else { block += v; v = 0; }
        }
        hbh_batches::File& F = B->files[o.tid / B->batch_size];
        std::string& s = F.pending;
        s += R->id[o.qid]; s += '\t'; s += std::to_string(o.qlen); s += '\t'; s += std::to_string(o.qstart); s += '\t';
        s += std::to_string(o.qend); s += '\t'; s += o.strand ? '-' : '+'; s += '\t'; s += R->id[o.tid]; s += '\t';
        s += std::to_string(o.tlen); s += '\t'; s += std::to_string(o.tstart); s += '\t'; s += std::to_string(o.tend); s += '\t';
        s += std::to_string(matches[i]); s += '\t'; s += std::to_string(block); s += '\t'; s.append((const char*)paf->buf.data() + paf->mapq[i].first, paf->mapq[i].second);
        s += "\tcg:Z:"; s.append((const char*)o.cigar, o.cigar_len); s += '\n';
        F.lines++;
        B->written++;
        if (s.size() >= (4u << 20) && !flush_batch(B, F, false)) return HB_ERR_INPUT;
    }
    return HB_OK;
}

// Finishes every file (frame end), frees `B`; lines_per_batch (may be NULL) receives each file's line count.
int hbh_batches_close(hbh_batches* B, uint64_t* lines_per_batch) {
    if (!B) return HB_ERR_ARG;
    int rc = HB_OK;
    for (size_t k = 0; k < B->files.size(); k++) {
        hbh_batches::File& F = B->files[k];
        if (F.f && F.cctx && rc == HB_OK && !flush_batch(B, F, true)) rc = HB_ERR_INPUT;  // ZSTD_e_end: the frame is complete
        if (F.cctx) zstd().freeCCtx(F.cctx);
        if (F.f && fclose(F.f) != 0 && rc == HB_OK) { t_err = "close failed"; rc = HB_ERR_INPUT; }
        if (lines_per_batch) lines_per_batch[k] = F.lines;
    }
    delete B;
    return rc;
}

// `herro align`: the FASTQ's reads (those of at least min_len bases) on device `device` in a context without weights, the PAF
// streamed through hb_align_overlaps chunk_lines lines at a time, the aligned lines written as hbh_batches_write writes them.
// times6: FASTQ load, context + upload, PAF read, alignment calls (wall), formatting + writing, total (s); counts7: lines read,
// skipped (unknown names, self overlaps), aligned and written, of those at the band's edge, failed (not written), cells, device ms.
int hbh_align(const char* reads_path, const char* paf_path, const char* out_dir, int device, uint32_t min_len, uint32_t band_w,
              uint32_t batch_size, uint32_t chunk_lines, int io_threads, double* times6, uint64_t* counts7) {
    if (!reads_path || !paf_path || !out_dir || !times6 || !counts7 || !chunk_lines) { t_err = "bad arguments"; return HB_ERR_ARG; }
    const double t_begin = now_s();
    std::fill(times6, times6 + 6, 0.0);
    std::fill(counts7, counts7 + 7, 0ull);
    hbh_reads* R = nullptr;
    int rc = hbh_reads_load(reads_path, min_len, nullptr, 0, nullptr, 0, io_threads, &R);
    if (rc) return rc;
    times6[0] = now_s() - t_begin;
    hb_ctx* ctx = nullptr;
    hbh_paf* P = nullptr;
    hbh_batches* B = nullptr;
    double ms_dev = 0;
    auto done = [&](int code) {
        if (code && ctx && t_err.empty()) t_err = hb_last_error(ctx);
        if (B) { const int c = hbh_batches_close(B, nullptr); if (!code) code = c; }
        if (P) hbh_paf_close(P);
        if (ctx) hb_destroy(ctx);
        hbh_reads_free(R);
        times6[5] = now_s() - t_begin;
        counts7[6] = (uint64_t)ms_dev;
        return code;
    };
    double t0 = now_s();
    hb_options opt{};
    opt.struct_size = sizeof opt; opt.window_size = std::max<uint32_t>(min_len, 1); opt.batch_size = 64; opt.flags = HB_FLAG_NO_MODEL;
    if (hb_create(&ctx, device, nullptr, &opt) != HB_OK) { t_err = std::string("hb_create: ") + hb_last_error(nullptr); ctx = nullptr; return done(HB_ERR_CUDA); }
    if (hb_upload_reads(ctx, hbh_reads_count(R), hbh_reads_word_ptrs(R), hbh_reads_lens(R), hbh_reads_qual_ptrs(R)) != HB_OK) {
        t_err = std::string("hb_upload_reads: ") + hb_last_error(ctx);
        return done(HB_ERR_CUDA);
    }
    times6[1] = now_s() - t0;
    if ((rc = hbh_paf_open(paf_path, R, &P))) return done(rc);
    if ((rc = hbh_batches_open(out_dir, R, batch_size, &B))) return done(rc);
    std::vector<hb_overlap> out;
    std::vector<uint8_t> text;
    std::vector<int32_t> status;
    std::vector<uint32_t> matches;
    for (;;) {
        t0 = now_s();
        uint32_t n = 0;
        if ((rc = hbh_paf_next(P, chunk_lines, &n))) return done(rc);
        times6[2] += now_s() - t0;
        if (!n) break;
        t0 = now_s();
        hb_align_shape sh{};
        if ((rc = hb_align_overlaps(ctx, n, hbh_paf_overlaps(P), band_w, &sh))) { t_err = std::string("hb_align_overlaps: ") + hb_last_error(ctx); return done(rc); }
        out.resize(n); text.resize(std::max<uint64_t>(sh.cigar_bytes, 1)); status.resize(n); matches.resize(n);
        if ((rc = hb_align_fetch(ctx, &sh, out.data(), text.data(), status.data(), matches.data()))) { t_err = hb_last_error(ctx); return done(rc); }
        times6[3] += now_s() - t0;
        ms_dev += sh.ms_device;
        counts7[4] += sh.n_failed;
        counts7[3] += sh.n_band_edge;
        counts7[2] += n - sh.n_failed;
        counts7[5] += sh.cells;
        t0 = now_s();
        if ((rc = hbh_batches_write(B, P, out.data(), status.data(), matches.data(), n))) return done(rc);
        times6[4] += now_s() - t0;
    }
    uint64_t c3[3];
    hbh_paf_stats(P, c3);
    counts7[0] = c3[0];
    counts7[1] = c3[1];
    t0 = now_s();
    rc = hbh_batches_close(B, nullptr);
    B = nullptr;
    times6[4] += now_s() - t0;
    return done(rc);
}

}  // extern "C"
