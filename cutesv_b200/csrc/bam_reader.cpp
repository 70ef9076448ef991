// bam_reader.cpp -- native BAM -> columnar packet decoder (host data loader, SURVEY 8f-3).
//
// Replaces the per-read Python loop over pysam objects (cuteSV:709-733) for plain BAM input: BGZF
// blocks are inflated by a small thread pool, records are parsed straight into the int32 columns /
// BAM-native u32 CIGAR array / reduced SA-segment table that csv_extract consumes (see
// include/cutesv_b200.h: csv_read_cols, csv_sa_cols).  No htslib: the BAM and BGZF layouts are
// implemented from the SAM/BAM specification.  Built as libcutesv_bam.so (g++ -lz -pthread).
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <zlib.h>

#include <algorithm>
#include <condition_variable>
#include <functional>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

namespace {

thread_local std::string g_err;

struct Block { std::vector<uint8_t> comp; uint8_t* dst; uint32_t isize; bool ok; };

bool inflate_block(Block& b) {
    if (b.isize == 0) return true;
    z_stream zs;
    memset(&zs, 0, sizeof(zs));
    if (inflateInit2(&zs, -15) != Z_OK) return false;
    zs.next_in = b.comp.data();
    zs.avail_in = (uInt)b.comp.size();
    zs.next_out = b.dst;
    zs.avail_out = (uInt)b.isize;
    int rc = inflate(&zs, Z_FINISH);
    inflateEnd(&zs);
    return rc == Z_STREAM_END && zs.total_out == b.isize;
}

// Decompressed bytes of one batch of BGZF blocks, inflated in place (no staging copy): [head, end) is valid
// data; the HEADROOM bytes in front of the payload receive the tail of a record that started in the previous
// chunk, so that every record is contiguous in exactly one chunk.
static constexpr size_t HEADROOM_DEFAULT = 4u << 20;
struct Chunk {
    std::unique_ptr<uint8_t[]> mem;
    uint8_t* head = nullptr;   // first valid byte
    uint8_t* end = nullptr;
};

// A batch of BGZF blocks being inflated by the pool.
struct Batch {
    std::vector<Block> blocks;
    std::unique_ptr<Chunk> chunk;
    size_t next = 0, done = 0;   // guarded by Pool::m
};

// Persistent inflate workers (threads that live as long as the reader: short-lived threads do not get
// spread over the cores quickly enough for 64 KB blocks).
struct Pool {
    std::vector<std::thread> th;
    std::mutex m;
    std::condition_variable cv_work, cv_done;
    Batch* cur = nullptr;
    bool stop = false;
    void start(int n) {
        for (int i = 0; i < n; i++) th.emplace_back([this]() { run(); });
    }
    void run() {
        std::unique_lock<std::mutex> lk(m);
        for (;;) {
            cv_work.wait(lk, [this]() { return stop || (cur && cur->next < cur->blocks.size()); });
            if (stop) return;
            Batch* b = cur;
            const size_t i = b->next++;
            lk.unlock();
            b->blocks[i].ok = inflate_block(b->blocks[i]);
            lk.lock();
            if (++b->done == b->blocks.size()) cv_done.notify_all();
        }
    }
    void submit(Batch* b) {
        { std::lock_guard<std::mutex> lk(m); cur = b; }
        cv_work.notify_all();
    }
    void wait(Batch* b) {
        std::unique_lock<std::mutex> lk(m);
        cv_done.wait(lk, [b]() { return b->done == b->blocks.size(); });
        if (cur == b) cur = nullptr;
    }
    ~Pool() {
        { std::lock_guard<std::mutex> lk(m); stop = true; }
        cv_work.notify_all();
        for (auto& t : th) t.join();
    }
};

// Persistent fork-join workers for the record parser: run(n, fn) calls fn(0..n-1) on the pool and returns
// when all are done.
struct ForkJoin {
    std::vector<std::thread> th;
    std::mutex m;
    std::condition_variable cv_work, cv_done;
    std::function<void(int)> fn;
    int n = 0, next = 0, done = 0;
    uint64_t epoch = 0;
    bool stop = false;
    void start(int k) { for (int i = 0; i < k; i++) th.emplace_back([this]() { loop(); }); }
    void loop() {
        std::unique_lock<std::mutex> lk(m);
        for (;;) {
            cv_work.wait(lk, [this]() { return stop || next < n; });
            if (stop) return;
            const int i = next++;
            lk.unlock();
            fn(i);
            lk.lock();
            if (++done == n) cv_done.notify_all();
        }
    }
    void run(int count, std::function<void(int)> f) {
        if (count <= 0) return;
        if (th.empty()) { for (int i = 0; i < count; i++) f(i); return; }
        std::unique_lock<std::mutex> lk(m);
        fn = std::move(f); n = count; next = 0; done = 0;
        cv_work.notify_all();
        cv_done.wait(lk, [this]() { return done == n; });
        n = 0; next = 0;
    }
    ~ForkJoin() {
        { std::lock_guard<std::mutex> lk(m); stop = true; }
        cv_work.notify_all();
        for (auto& t : th) t.join();
    }
};

// variable-length output of one parser task (a contiguous range of records)
struct ThreadOut {   // (CIGAR and sequence sizes are known from the fixed fields: those go straight to their final place)
    std::vector<int32_t> sa_chrom, sa_pos0, sa_strand, sa_mapq, sa_first, sa_last, sa_span;
    void clear() { sa_chrom.clear(); sa_pos0.clear(); sa_strand.clear(); sa_mapq.clear(); sa_first.clear(); sa_last.clear(); sa_span.clear(); }
};

struct Reader {
    FILE* f = nullptr;
    bool eof = false;            // no more blocks in the file
    std::vector<std::unique_ptr<Chunk>> chunks;   // chunks holding records of the packet being built; back() is current
    const uint8_t* cur = nullptr;                 // read position inside chunks.back()
    int n_threads = 4;
    int batch_blocks = 256;              // BGZF blocks per chunk
    size_t headroom = HEADROOM_DEFAULT;
    // (declared BEFORE the pools: members are destroyed in reverse order, so the workers are joined before the
    //  blocks / chunk they inflate into are freed)
    Batch batch[2];              // [inflight] is being inflated while the parser consumes the other's payload
    int inflight = -1;
    Pool pool;
    ForkJoin parsers;
    std::vector<ThreadOut> touts;
    std::vector<const uint8_t*> rec_ptr;   // start of every record of the packet being built
    std::string io_err;          // error met while reading ahead (reported when that batch is consumed)
    // header
    std::vector<std::string> ref_name;
    std::vector<int64_t> ref_len;
    std::vector<int32_t> chrom_id;   // header index -> contig id handed to the kernels
    std::unordered_map<std::string, int32_t> ref_index;
    // read names -> provisional ids (first-seen order)
    std::unordered_map<std::string, int32_t> name_id;
    std::vector<std::string> names;
    // packet storage (valid until the next bamr_next)
    std::vector<int32_t> chrom, ref_start, ref_end, flag, mapq, query_len, read_id;
    std::vector<int64_t> cigar_off, sa_off, seq_off;
    std::vector<uint32_t> cigar;
    std::vector<int32_t> sa_chrom, sa_pos0, sa_strand, sa_mapq, sa_first, sa_last, sa_span;
    std::vector<uint8_t> seq4;
    bool keep_seq = true;
};

// read up to `max_blocks` raw BGZF blocks from the file into `b`; false + r.io_err on a malformed file
bool read_blocks(Reader& r, Batch& b, int max_blocks) {
    b.blocks.clear();
    b.next = b.done = 0;
    for (int i = 0; i < max_blocks && !r.eof; i++) {
        uint8_t h[18];
        size_t got = fread(h, 1, 18, r.f);
        if (got == 0) { r.eof = true; break; }
        if (got != 18 || h[0] != 31 || h[1] != 139 || h[2] != 8 || !(h[3] & 4)) { r.io_err = got == 18 ? "not a BGZF block" : "truncated BGZF header"; return false; }
        const int xlen = h[10] | (h[11] << 8);
        int bsize = -1;
        std::vector<uint8_t> extra(xlen);
        memcpy(extra.data(), h + 12, std::min(6, xlen));
        if (xlen > 6 && fread(extra.data() + 6, 1, xlen - 6, r.f) != (size_t)(xlen - 6)) { r.io_err = "truncated BGZF header"; return false; }
        for (int o = 0; o + 4 <= xlen;) {
            const int slen = extra[o + 2] | (extra[o + 3] << 8);
            if (extra[o] == 'B' && extra[o + 1] == 'C' && slen == 2 && o + 6 <= xlen) bsize = extra[o + 4] | (extra[o + 5] << 8);
            o += 4 + slen;
        }
        if (bsize < 0) { r.io_err = "BGZF block without BC field"; return false; }
        const int clen = bsize + 1 - 12 - xlen - 8;  // deflate payload length
        Block blk;
        blk.comp.resize(clen > 0 ? clen : 0);
        uint8_t tail[8];
        if ((clen > 0 && fread(blk.comp.data(), 1, clen, r.f) != (size_t)clen) || fread(tail, 1, 8, r.f) != 8) { r.io_err = "truncated BGZF block"; return false; }
        blk.isize = tail[4] | (tail[5] << 8) | (tail[6] << 16) | ((uint32_t)tail[7] << 24);
        if (blk.isize > 65536u) { r.io_err = "BGZF block larger than 64 KiB"; return false; }   // SAM spec 4.1
        blk.ok = true;
        b.blocks.push_back(std::move(blk));
    }
    return true;
}

// start inflating the next batch of the file (if any) in the background
void prefetch(Reader& r) {
    if (r.inflight >= 0 || r.eof || !r.io_err.empty()) return;
    Batch& b = r.batch[0];
    read_blocks(r, b, r.batch_blocks);
    if (b.blocks.empty()) return;
    size_t total = 0;
    for (auto& blk : b.blocks) total += blk.isize;
    b.chunk.reset(new Chunk());
    b.chunk->mem.reset(new uint8_t[r.headroom + total]);   // uninitialised on purpose
    b.chunk->head = b.chunk->mem.get() + r.headroom;
    b.chunk->end = b.chunk->head + total;
    uint8_t* o = b.chunk->head;
    for (auto& blk : b.blocks) { blk.dst = o; o += blk.isize; }
    r.inflight = 0;
    r.pool.submit(&b);
}

// Makes the next chunk current, carrying the unread tail of the present one in front of it.
// 1 ok, 0 clean end of file (nothing more to read), -1 error (g_err set).
int next_chunk(Reader& r) {
    if (r.inflight < 0) prefetch(r);
    if (r.inflight < 0) {
        if (!r.io_err.empty()) { g_err = r.io_err; return -1; }
        return 0;
    }
    Batch& b = r.batch[r.inflight];
    r.pool.wait(&b);
    for (auto& blk : b.blocks)
        if (!blk.ok) { g_err = "BGZF inflate failed"; return -1; }
    std::unique_ptr<Chunk> c = std::move(b.chunk);
    r.inflight = -1;
    const size_t carry = r.chunks.empty() ? 0 : (size_t)(r.chunks.back()->end - r.cur);
    if (carry > (size_t)(c->head - c->mem.get())) {  // a record larger than the headroom: rebuild the chunk with room for it (rare)
        const size_t total = (size_t)(c->end - c->head);
        std::unique_ptr<Chunk> big(new Chunk());
        big->mem.reset(new uint8_t[carry + total]);
        big->head = big->mem.get() + carry;
        big->end = big->head + total;
        memcpy(big->head, c->head, total);
        c = std::move(big);
    }
    if (carry) {
        memcpy(c->head - carry, r.cur, carry);
        c->head -= carry;
        r.chunks.back()->end = const_cast<uint8_t*>(r.cur);   // those bytes now live in the new chunk
    }
    r.cur = c->head;
    r.chunks.push_back(std::move(c));
    prefetch(r);   // the following batch inflates while the caller works on this one
    return 1;
}

// `need` contiguous bytes at r.cur?  1 yes, 0 clean end of file, -1 error (g_err set)
int ensure(Reader& r, size_t need) {
    while (r.chunks.empty() || (size_t)(r.chunks.back()->end - r.cur) < need) {
        g_err.clear();
        const int st = next_chunk(r);
        if (st <= 0) return st;
    }
    return 1;
}

inline int32_t rd_i32(const uint8_t* p) { int32_t v; memcpy(&v, p, 4); return v; }
inline uint32_t rd_u32(const uint8_t* p) { uint32_t v; memcpy(&v, p, 4); return v; }
inline uint16_t rd_u16(const uint8_t* p) { uint16_t v; memcpy(&v, p, 2); return v; }

// (first S length, last S length, reference span) of a CIGAR string: acquire_clip_pos, cuteSV:466-481
void clip_pos(const char* s, size_t n, int32_t* first, int32_t* last, int32_t* span) {
    *first = 0; *last = 0; *span = 0;
    int64_t num = 0;
    bool first_op = true;
    int32_t last_len = 0;
    char last_op = 0;
    for (size_t i = 0; i < n; i++) {
        const char c = s[i];
        if (c >= '0' && c <= '9') { num = num * 10 + (c - '0'); continue; }
        if (first_op) { if (c == 'S') *first = (int32_t)num; first_op = false; }
        if (c == 'M' || c == 'D' || c == '=' || c == 'X') *span += (int32_t)num;
        last_len = (int32_t)num; last_op = c;
        num = 0;
    }
    if (last_op == 'S') *last = last_len;
}

size_t aux_skip(const uint8_t* p, const uint8_t* end, char type) {
    switch (type) {
        case 'A': case 'c': case 'C': return 1;
        case 's': case 'S': return 2;
        case 'i': case 'I': case 'f': return 4;
        case 'Z': case 'H': { size_t n = 0; while (p + n < end && p[n]) n++; return n + 1; }
        case 'B': {
            if (p + 5 > end) return (size_t)(end - p);
            const char st = (char)p[0];
            const uint32_t cnt = rd_u32(p + 1);
            const size_t es = (st == 'c' || st == 'C') ? 1 : (st == 's' || st == 'S') ? 2 : 4;
            return 5 + es * cnt;
        }
        default: return (size_t)(end - p);
    }
}

}  // namespace

extern "C" {

typedef struct bamr_packet {
    int64_t n;
    int32_t *chrom, *ref_start, *ref_end, *flag, *mapq, *query_len, *read_id;
    int64_t *cigar_off, *sa_off;
    int64_t n_cigar;
    uint32_t* cigar;
    int64_t n_sa;
    int32_t *sa_chrom, *sa_pos0, *sa_strand, *sa_mapq, *sa_first, *sa_last, *sa_span;
    int64_t* seq_off;
    uint8_t* seq4;
} bamr_packet;

const char* bamr_error(void) { return g_err.c_str(); }

static int bamr_open_impl(const char* path, int n_threads, void** out) {
    Reader* r = new Reader();
    r->f = fopen(path, "rb");
    if (!r->f) { g_err = std::string("cannot open ") + path; delete r; return -1; }
    r->n_threads = n_threads > 0 ? n_threads : 4;
    r->pool.start(r->n_threads);
    if (r->n_threads > 1) r->parsers.start(r->n_threads);
    g_err.clear();
    auto fail = [&](const char* msg) {
        if (g_err.empty()) g_err = msg;
        if (r->inflight >= 0) { r->pool.wait(&r->batch[r->inflight]); r->inflight = -1; }   // a read-ahead batch may still be inflating
        fclose(r->f); r->f = nullptr; delete r; return -1;
    };
    if (ensure(*r, 12) <= 0 || memcmp(r->cur, "BAM\1", 4) != 0) return fail("not a BAM file");
    const int32_t l_text = rd_i32(r->cur + 4);
    if (l_text < 0 || ensure(*r, 12 + (size_t)l_text) <= 0) return fail("truncated BAM header");
    r->cur += 8 + (size_t)l_text;
    const int32_t n_ref = rd_i32(r->cur);
    r->cur += 4;
    for (int32_t i = 0; i < n_ref; i++) {
        if (ensure(*r, 4) <= 0) return fail("truncated BAM header");
        const int32_t l_name = rd_i32(r->cur);
        if (l_name < 1 || ensure(*r, 4 + (size_t)l_name + 4) <= 0) return fail("truncated BAM header");
        std::string nm((const char*)r->cur + 4, (size_t)l_name - 1);
        const int32_t l_ref = rd_i32(r->cur + 4 + l_name);
        r->cur += 8 + (size_t)l_name;
        r->ref_index[nm] = i;
        r->ref_name.push_back(nm);
        r->ref_len.push_back(l_ref);
        r->chrom_id.push_back(i);
    }
    *out = r;
    return 0;
}

void bamr_close(void* h) {
    Reader* r = (Reader*)h;
    if (!r) return;
    if (r->inflight >= 0) { r->pool.wait(&r->batch[r->inflight]); r->inflight = -1; }   // closing before EOF: drain the read-ahead
    if (r->f) fclose(r->f);
    delete r;
}

int32_t bamr_n_ref(void* h) { return (int32_t)((Reader*)h)->ref_name.size(); }
const char* bamr_ref_name(void* h, int32_t i) { return ((Reader*)h)->ref_name[i].c_str(); }
int64_t bamr_ref_len(void* h, int32_t i) { return ((Reader*)h)->ref_len[i]; }
void bamr_set_chrom_ids(void* h, const int32_t* ids) { Reader* r = (Reader*)h; for (size_t i = 0; i < r->chrom_id.size(); i++) r->chrom_id[i] = ids[i]; }
void bamr_keep_seq(void* h, int keep) { ((Reader*)h)->keep_seq = keep != 0; }
// tests: BGZF blocks per chunk and the carry-over headroom (takes effect from the next chunk that is read)
void bamr_tune(void* h, int batch_blocks, int64_t headroom) {
    Reader* r = (Reader*)h;
    if (batch_blocks > 0) r->batch_blocks = batch_blocks;
    if (headroom >= 0) r->headroom = (size_t)headroom;
}

// SA:Z and the long-CIGAR CG:B,I tag of a record (p = first byte after block_size)
static void find_tags(const uint8_t* p, const uint8_t* end, const char** sa, const uint8_t** cg_tag, uint32_t* cg_cnt) {
    const int l_read_name = p[8];
    const int n_cigar = rd_u16(p + 12);
    const int32_t l_seq = rd_i32(p + 16);
    const uint8_t* aux = p + 32 + l_read_name + 4 * (size_t)n_cigar + (size_t)(l_seq + 1) / 2 + (size_t)l_seq;
    *sa = nullptr; *cg_tag = nullptr; *cg_cnt = 0;
    for (const uint8_t* a = aux; a + 3 <= end;) {
        const char t0 = (char)a[0], t1 = (char)a[1], ty = (char)a[2];
        const uint8_t* v = a + 3;
        if (t0 == 'S' && t1 == 'A' && ty == 'Z') *sa = (const char*)v;
        if (t0 == 'C' && t1 == 'G' && ty == 'B' && v + 5 <= end && (v[0] == 'I' || v[0] == 'i') && v + 5 + 4 * (size_t)rd_u32(v + 1) <= end) {
            *cg_cnt = rd_u32(v + 1); *cg_tag = v + 5;
        }
        a = v + aux_skip(v, end, ty);
    }
}
// a 2-op CIGAR "<l_seq>S<span>N" announces the real CIGAR in the CG tag (alignments with > 65535 ops)
static inline bool cg_placeholder(const uint8_t* cg, int n_cigar, int32_t l_seq) {
    return n_cigar == 2 && (rd_u32(cg) & 15) == 4 && (int32_t)(rd_u32(cg) >> 4) == l_seq && (rd_u32(cg + 4) & 15) == 3;
}

// Parses records [lo, hi) of r.rec_ptr: fixed-width fields straight into the packet columns (sized by the
// caller), variable-length parts into `o`; per-record lengths go to cigar_off / sa_off / seq_off [k + 1].
static void parse_range(Reader& r, size_t lo, size_t hi, ThreadOut& o) {
    o.clear();
    for (size_t k = lo; k < hi; k++) {
        const uint8_t* p = r.rec_ptr[k] + 4;
        const int32_t block_size = rd_i32(p - 4);
        const uint8_t* end = p + block_size;
        const int32_t ref_id = rd_i32(p), pos = rd_i32(p + 4);
        const int l_read_name = p[8], mq = p[9];
        const int n_cigar = rd_u16(p + 12), flg = rd_u16(p + 14);
        const int32_t l_seq = rd_i32(p + 16);
        const uint8_t* cg = p + 32 + l_read_name;
        const uint8_t* sq = cg + 4 * (size_t)n_cigar;
        const char* sa;
        const uint8_t* cg_tag;
        uint32_t cg_cnt;
        find_tags(p, end, &sa, &cg_tag, &cg_cnt);
        const uint8_t* cig_src = cg;
        uint32_t cig_n = (uint32_t)n_cigar;
        if (cg_tag && cg_placeholder(cg, n_cigar, l_seq)) { cig_src = cg_tag; cig_n = cg_cnt; }
        int32_t span = 0;
        uint32_t* cdst = r.cigar.data() + r.cigar_off[k];   // offsets were fixed by the scan phase
        for (uint32_t j = 0; j < cig_n; j++) {
            const uint32_t c = rd_u32(cig_src + 4 * (size_t)j);
            cdst[j] = c;
            const int op = c & 15;
            if (op == 0 || op == 2 || op == 3 || op == 7 || op == 8) span += (int32_t)(c >> 4);
        }
        r.chrom[k] = r.chrom_id[ref_id]; r.ref_start[k] = pos; r.ref_end[k] = pos + span; r.flag[k] = flg;
        r.mapq[k] = mq; r.query_len[k] = l_seq;
        const size_t s0 = o.sa_chrom.size();
        if (sa) {  // "rname,pos,strand,CIGAR,mapQ,NM;" ... (cuteSV:489-509)
            const char* s = sa;
            const char* lim = (const char*)end;   // never past the record, whether or not the NUL is there
            while (s < lim && *s) {
                const char* e = s;
                while (e < lim && *e && *e != ';') e++;
                const bool closed = e < lim && *e == ';';   // the reference keeps split(';')[:-1]: an entry without ';' is dropped (cuteSV:678)
                const char* f[6]; int nf = 0; f[nf++] = s;
                for (const char* q = s; q < e && nf < 6; q++) if (*q == ',') f[nf++] = q + 1;
                if (closed && nf >= 5) {
                    std::string rn(f[0], (size_t)(f[1] - f[0] - 1));
                    auto ri = r.ref_index.find(rn);
                    int32_t fc, lc, sp;
                    clip_pos(f[3], (size_t)(f[4] - f[3] - 1), &fc, &lc, &sp);
                    o.sa_chrom.push_back(ri == r.ref_index.end() ? -1 : r.chrom_id[ri->second]);
                    o.sa_pos0.push_back(atoi(f[1]) - 1);
                    o.sa_strand.push_back(*f[2] == '+' ? 0 : 1);
                    o.sa_mapq.push_back(atoi(f[4]));
                    o.sa_first.push_back(fc); o.sa_last.push_back(lc); o.sa_span.push_back(sp);
                }
                s = closed ? e + 1 : e;
                if (!closed) break;
            }
        }
        r.sa_off[k + 1] = (int64_t)(o.sa_chrom.size() - s0);
        if (r.keep_seq && l_seq > 0) memcpy(r.seq4.data() + r.seq_off[k], sq, (size_t)(l_seq + 1) / 2);
    }
}

// Next packet of up to max_records MAPPED records (file order).  Returns the record count (0 at EOF,
// -1 on error); pointers stay valid until the next call.
// Three phases: (1) sequential hop over the block_size chain + read-name ids (first-seen order), (2) the
// records are parsed by the fork-join pool in contiguous ranges, (3) the variable-length parts are stitched.
static int64_t bamr_next_impl(void* h, int64_t max_records, bamr_packet* out) {
    Reader& r = *(Reader*)h;
    r.rec_ptr.clear();
    r.read_id.clear();
    r.cigar_off.assign(1, 0); r.seq_off.assign(1, 0);
    if (r.chunks.size() > 1) r.chunks.erase(r.chunks.begin(), r.chunks.end() - 1);   // the previous packet's chunks
    while ((int64_t)r.rec_ptr.size() < max_records) {
        int st = ensure(r, 4);
        if (st < 0) return -1;
        if (st == 0) {
            if (!r.chunks.empty() && r.chunks.back()->end > r.cur) { g_err = "truncated BAM record"; return -1; }
            break;
        }
        const int32_t block_size = rd_i32(r.cur);
        if (block_size < 32) { g_err = "corrupt BAM record"; return -1; }
        st = ensure(r, 4 + (size_t)block_size);
        if (st <= 0) { if (st == 0) g_err = "truncated BAM record"; return -1; }
        const uint8_t* rec = r.cur;
        const uint8_t* p = rec + 4;
        const int32_t ref_id = rd_i32(p);
        r.cur += 4 + (size_t)block_size;
        if (ref_id < 0 || ref_id >= (int32_t)r.ref_name.size()) continue;  // unmapped / unplaced: never returned by fetch(chr, ...)
        const int l_read_name = p[8];
        {   // the fixed-size fields must describe a record that fits its block_size (the parser trusts them)
            const int64_t n_cig = rd_u16(p + 12), l_seq = rd_i32(p + 16);
            if (l_seq < 0 || 32 + (int64_t)l_read_name + 4 * n_cig + (l_seq + 1) / 2 + l_seq > (int64_t)block_size) {
                g_err = "corrupt BAM record";
                return -1;
            }
        }
        std::string name((const char*)p + 32, (size_t)(l_read_name > 0 ? l_read_name - 1 : 0));
        auto it = r.name_id.find(name);
        int32_t id;
        if (it == r.name_id.end()) { id = (int32_t)r.names.size(); r.name_id.emplace(name, id); r.names.push_back(std::move(name)); }
        else id = it->second;
        {   // sizes of the variable-length parts that the fixed fields (or, rarely, the CG tag) already tell
            const int n_cig = rd_u16(p + 12);
            const int32_t l_seq = rd_i32(p + 16);
            int64_t cig_n = n_cig;
            const uint8_t* cg = p + 32 + l_read_name;
            if (cg_placeholder(cg, n_cig, l_seq)) {
                const char* sa; const uint8_t* cg_tag; uint32_t cg_cnt;
                find_tags(p, p + block_size, &sa, &cg_tag, &cg_cnt);
                if (cg_tag) cig_n = cg_cnt;
            }
            r.cigar_off.push_back(r.cigar_off.back() + cig_n);
            r.seq_off.push_back(r.seq_off.back() + (r.keep_seq ? (int64_t)((l_seq + 1) / 2) : 0));
        }
        r.rec_ptr.push_back(rec);
        r.read_id.push_back(id);
    }
    const size_t n = r.rec_ptr.size();
    r.chrom.resize(n); r.ref_start.resize(n); r.ref_end.resize(n); r.flag.resize(n); r.mapq.resize(n); r.query_len.resize(n);
    r.sa_off.assign(n + 1, 0);
    r.cigar.resize((size_t)r.cigar_off[n]); r.seq4.resize((size_t)r.seq_off[n]);
    const int T = (int)std::max<size_t>(1, std::min<size_t>((size_t)r.n_threads * 4, (n + 255) / 256));
    if (r.touts.size() < (size_t)T) r.touts.resize((size_t)T);
    auto range = [&](int t) { return std::make_pair(n * (size_t)t / (size_t)T, n * (size_t)(t + 1) / (size_t)T); };
    r.parsers.run(T, [&](int t) { auto rg = range(t); parse_range(r, rg.first, rg.second, r.touts[(size_t)t]); });
    // stitch: per-record lengths -> offsets; per-task blocks -> one array each
    for (size_t k = 0; k < n; k++) r.sa_off[k + 1] += r.sa_off[k];
    const size_t ns = n ? (size_t)r.sa_off[n] : 0;
    r.sa_chrom.resize(ns); r.sa_pos0.resize(ns); r.sa_strand.resize(ns); r.sa_mapq.resize(ns); r.sa_first.resize(ns); r.sa_last.resize(ns); r.sa_span.resize(ns);
    r.parsers.run(T, [&](int t) {
        auto rg = range(t);
        if (rg.first == rg.second) return;
        const ThreadOut& o = r.touts[(size_t)t];
        const size_t s0 = (size_t)r.sa_off[rg.first];
        if (!o.sa_chrom.empty()) {
            const size_t b = o.sa_chrom.size() * 4;
            memcpy(r.sa_chrom.data() + s0, o.sa_chrom.data(), b); memcpy(r.sa_pos0.data() + s0, o.sa_pos0.data(), b);
            memcpy(r.sa_strand.data() + s0, o.sa_strand.data(), b); memcpy(r.sa_mapq.data() + s0, o.sa_mapq.data(), b);
            memcpy(r.sa_first.data() + s0, o.sa_first.data(), b); memcpy(r.sa_last.data() + s0, o.sa_last.data(), b);
            memcpy(r.sa_span.data() + s0, o.sa_span.data(), b);
        }
    });
    out->n = (int64_t)n;
    out->chrom = r.chrom.data(); out->ref_start = r.ref_start.data(); out->ref_end = r.ref_end.data(); out->flag = r.flag.data();
    out->mapq = r.mapq.data(); out->query_len = r.query_len.data(); out->read_id = r.read_id.data();
    out->cigar_off = r.cigar_off.data(); out->sa_off = r.sa_off.data();
    out->n_cigar = (int64_t)r.cigar.size(); out->cigar = r.cigar.data();
    out->n_sa = (int64_t)r.sa_chrom.size();
    out->sa_chrom = r.sa_chrom.data(); out->sa_pos0 = r.sa_pos0.data(); out->sa_strand = r.sa_strand.data(); out->sa_mapq = r.sa_mapq.data();
    out->sa_first = r.sa_first.data(); out->sa_last = r.sa_last.data(); out->sa_span = r.sa_span.data();
    out->seq_off = r.seq_off.data(); out->seq4 = r.seq4.data();
    return (int64_t)n;
}

int64_t bamr_n_names(void* h) { return (int64_t)((Reader*)h)->names.size(); }
const char* bamr_name(void* h, int64_t id) { return ((Reader*)h)->names[(size_t)id].c_str(); }
// rank[provisional id] = rank of the name in byte-wise (== Python str for ASCII) order
void bamr_name_ranks(void* h, int32_t* rank) {
    Reader& r = *(Reader*)h;
    std::vector<int32_t> order(r.names.size());
    for (size_t i = 0; i < order.size(); i++) order[i] = (int32_t)i;
    std::sort(order.begin(), order.end(), [&](int32_t a, int32_t b) { return r.names[a] < r.names[b]; });
    for (size_t i = 0; i < order.size(); i++) rank[order[i]] = (int32_t)i;
}
// 4-bit packed -> ASCII
void bamr_decode_seq(const uint8_t* seq4, int64_t l_seq, char* out) {
    static const char tab[] = "=ACMGRSVTWYHKDBN";
    for (int64_t i = 0; i < l_seq; i++) out[i] = tab[(seq4[i >> 1] >> ((~i & 1) << 2)) & 15];
}

// many base ranges at once: range i = `len[i]` bases starting at nibble `nib0[i]` of seq4, written as ASCII at out + out_off[i]
// (the INS signature sequences of a whole packet, cutesv_b200/packing.py::ins_block_from_packed)
void bamr_unpack_ranges(const uint8_t* seq4, int64_t n, const int64_t* nib0, const int64_t* len, const int64_t* out_off, char* out) {
    static const char tab[] = "=ACMGRSVTWYHKDBN";
    for (int64_t i = 0; i < n; i++) {
        char* o = out + out_off[i];
        const int64_t s = nib0[i];
        for (int64_t k = 0; k < len[i]; k++) o[k] = tab[(seq4[(s + k) >> 1] >> ((~(s + k) & 1) << 2)) & 15];
    }
}

// The same counts from a CSI index (`samtools index -c`, needed for contigs longer than 2^29 bp). The file is BGZF
// compressed: magic, min_shift, depth, l_aux, aux, n_ref; per reference n_bin bins of (bin, loffset, n_chunk, chunks) and
// no linear index. The pseudo-bin is ((1 << 3*(depth+1)) - 1)/7 + 1; its second chunk holds (n_mapped, n_unmapped).
static int csi_stats(const char* path, int32_t n_ref, int64_t* mapped) {
    gzFile f = gzopen(path, "rb");
    if (!f) { g_err = std::string("cannot open ") + path; return -1; }
    std::vector<uint8_t> d;
    std::vector<uint8_t> buf(1 << 16);
    int k;
    while ((k = gzread(f, buf.data(), (unsigned)buf.size())) > 0) d.insert(d.end(), buf.begin(), buf.begin() + k);
    int zerr = Z_OK;
    gzerror(f, &zerr);
    gzclose(f);
    if (k < 0 || (zerr != Z_OK && zerr != Z_STREAM_END)) { g_err = "truncated or corrupt CSI (BGZF decompression failed)"; return -1; }
    size_t p = 0;
    auto have = [&](uint64_t b) { return b <= d.size() - p; };
    if (!have(16) || memcmp(d.data(), "CSI\1", 4) != 0) { g_err = "not a CSI index"; return -1; }
    const int32_t min_shift = rd_i32(d.data() + 4), depth = rd_i32(d.data() + 8), l_aux = rd_i32(d.data() + 12);
    if (min_shift < 0 || depth < 0 || depth > 10) { g_err = "malformed CSI (min_shift / depth)"; return -1; }
    p = 16;
    if (l_aux < 0 || !have((uint64_t)l_aux + 4)) { g_err = "truncated CSI (header)"; return -1; }
    p += (size_t)l_aux;
    const int32_t n = rd_i32(d.data() + p);
    p += 4;
    if (n < 0) { g_err = "malformed CSI (negative reference count)"; return -1; }
    const uint32_t pseudo = (uint32_t)((((uint64_t)1 << (3 * (depth + 1))) - 1) / 7 + 1);
    for (int32_t i = 0; i < n_ref; i++) mapped[i] = 0;
    for (int32_t ref = 0; ref < n; ref++) {
        if (!have(4)) { g_err = "truncated CSI"; return -1; }
        const int32_t n_bin = rd_i32(d.data() + p);
        p += 4;
        if (n_bin < 0) { g_err = "malformed CSI (negative bin count)"; return -1; }
        for (int32_t b = 0; b < n_bin; b++) {
            if (!have(16)) { g_err = "truncated CSI"; return -1; }
            const uint32_t bin = rd_u32(d.data() + p);
            const int32_t n_chunk = rd_i32(d.data() + p + 12);   // after bin (4 B) and loffset (8 B)
            p += 16;
            if (n_chunk < 0) { g_err = "malformed CSI (chunk count)"; return -1; }
            if (!have((uint64_t)n_chunk * 16)) { g_err = "truncated CSI"; return -1; }
            if (bin == pseudo && n_chunk >= 2 && ref < n_ref) { uint64_t m; memcpy(&m, d.data() + p + 16, 8); mapped[ref] = (int64_t)m; }
            p += (size_t)n_chunk * 16;
        }
    }
    return 0;
}

// Per-reference mapped-read counts from a .bai index (get_index_statistics, cuteSV:1015-1025):
// the pseudo-bin 37450 of every reference holds (n_mapped, n_unmapped).  A BGZF-compressed file is read as CSI.
static int bamr_index_stats_impl(const char* bai_path, int32_t n_ref, int64_t* mapped) {
    FILE* f = fopen(bai_path, "rb");
    if (!f) { g_err = std::string("cannot open ") + bai_path; return -1; }
    uint8_t h[8];
    const size_t got = fread(h, 1, 8, f);
    if (got >= 2 && h[0] == 31 && h[1] == 139) { fclose(f); return csi_stats(bai_path, n_ref, mapped); }
    if (got != 8 || memcmp(h, "BAI\1", 4) != 0) { fclose(f); g_err = "not a BAI index"; return -1; }
    const int32_t n = rd_i32(h + 4);
    for (int32_t i = 0; i < n_ref; i++) mapped[i] = 0;
    for (int32_t ref = 0; ref < n; ref++) {
        uint8_t b4[4];
        if (fread(b4, 1, 4, f) != 4) break;
        const int32_t n_bin = rd_i32(b4);
        if (n_bin < 0) { fclose(f); g_err = "malformed BAI (negative bin count)"; return -1; }
        for (int32_t b = 0; b < n_bin; b++) {
            uint8_t bh[8];
            if (fread(bh, 1, 8, f) != 8) { fclose(f); g_err = "truncated BAI"; return -1; }
            const uint32_t bin = rd_u32(bh);
            const int32_t n_chunk = rd_i32(bh + 4);
            if (n_chunk < 0 || n_chunk > (1 << 26)) { fclose(f); g_err = "malformed BAI (chunk count)"; return -1; }
            std::vector<uint8_t> ch((size_t)n_chunk * 16);
            if (n_chunk && fread(ch.data(), 1, ch.size(), f) != ch.size()) { fclose(f); g_err = "truncated BAI"; return -1; }
            if (bin == 37450 && n_chunk >= 2 && ref < n_ref) { uint64_t m; memcpy(&m, ch.data() + 16, 8); mapped[ref] = (int64_t)m; }
        }
        if (fread(b4, 1, 4, f) != 4) break;
        const int32_t n_intv = rd_i32(b4);
        if (n_intv && fseek(f, (long)n_intv * 8, SEEK_CUR) != 0) break;
    }
    fclose(f);
    return 0;
}

// No exception crosses the C boundary (std::bad_alloc on a malformed file, ...): error text in bamr_error().
int bamr_open(const char* path, int n_threads, void** out) {
    try { return bamr_open_impl(path, n_threads, out); } catch (const std::exception& e) { g_err = std::string("bamr_open: ") + e.what(); return -1; } catch (...) { g_err = "bamr_open: unknown error"; return -1; }
}
int64_t bamr_next(void* h, int64_t max_records, bamr_packet* out) {
    try { return bamr_next_impl(h, max_records, out); } catch (const std::exception& e) { g_err = std::string("bamr_next: ") + e.what(); return -1; } catch (...) { g_err = "bamr_next: unknown error"; return -1; }
}
int bamr_index_stats(const char* bai_path, int32_t n_ref, int64_t* mapped) {
    try { return bamr_index_stats_impl(bai_path, n_ref, mapped); } catch (const std::exception& e) { g_err = std::string("bamr_index_stats: ") + e.what(); return -1; } catch (...) { g_err = "bamr_index_stats: unknown error"; return -1; }
}

}  // extern "C"
