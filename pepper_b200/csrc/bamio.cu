// Host-side BAM / BGZF / BAI and FASTA / FAI readers (SURVEY 8f row f4): the file I/O under BAM_handler / FASTA_handler
// (pepper/modules/src/dataio/bam_handler.cpp:6-28,115-135, fasta_handler.cpp:7-55), which the reference gets from
// htslib 1.9 (sam_open / sam_index_load / sam_hdr_read / sam_itr_queryi / sam_itr_next, fai_load / faidx_fetch_seq).
// Written from the format specification (SAMv1 4.1 BGZF, 4.2 BAM, 5.2 BAI; faidx 5-column index), not from htslib.
//
// pb_bam_fetch hands back every record the htslib iterator would return for (tid, beg, end) - file order, overlap rule
// pos < end && pos + max(rlen, n_cigar ? 0 : 1) > beg - as a pb_records_t in (page-locked when a GPU is present) host
// memory, ready for pb_get_reads_plan_host / one cudaMemcpy.  BGZF blocks of a fetch are inflated by a thread pool and
// the records are scattered into the SoA arrays in parallel; the trim itself runs on the GPU (get_reads.cu).
// pb_bam_fetch is host plumbing (thread-pool zlib inflate); pb_bam_fetch_device is the GPU path: the host only selects the BGZF
// blocks (index arithmetic + block headers) and copies their COMPRESSED bytes; inflate, record walk, parse and the SoA
// scatter are kernels (bgzf_inflate.cuh) and the records never visit host memory.
#include "common.cuh"
#include "bgzf_inflate.cuh"
#include <zlib.h>
#include <fcntl.h>
#include <sched.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>
#include <algorithm>
#include <atomic>
#include <map>
#include <string>
#include <thread>
#include <vector>
#include <chrono>
#include <condition_variable>
#include <functional>
#include <mutex>

using namespace pb;

namespace {

struct MappedFile {
    const uint8_t *p = nullptr;
    size_t n = 0;
    int fd = -1;
    bool open(const char *path) {
        fd = ::open(path, O_RDONLY);
        if (fd < 0) return false;
        struct stat st;
        if (fstat(fd, &st) != 0) { ::close(fd); fd = -1; return false; }
        n = (size_t) st.st_size;
        if (n == 0) { p = nullptr; return true; }
        void *m = mmap(nullptr, n, PROT_READ, MAP_PRIVATE, fd, 0);
        if (m == MAP_FAILED) { ::close(fd); fd = -1; return false; }
        p = (const uint8_t *) m;
        return true;
    }
    void close() {
        if (p) munmap((void *) p, n);
        if (fd >= 0) ::close(fd);
        p = nullptr; fd = -1; n = 0;
    }
};

inline uint16_t rd16(const uint8_t *p) { uint16_t v; memcpy(&v, p, 2); return v; }
inline uint32_t rd32(const uint8_t *p) { uint32_t v; memcpy(&v, p, 4); return v; }
inline int32_t rdi32(const uint8_t *p) { int32_t v; memcpy(&v, p, 4); return v; }
inline uint64_t rd64(const uint8_t *p) { uint64_t v; memcpy(&v, p, 8); return v; }

// size of the BGZF block at `off` (0 when it is not a valid block header); payload offset returned through *data_off
size_t bgzf_block_size(const uint8_t *f, size_t n, size_t off, size_t *data_off) {
    if (off + 18 > n) return 0;
    const uint8_t *h = f + off;
    if (h[0] != 0x1f || h[1] != 0x8b || h[2] != 8 || !(h[3] & 4)) return 0;
    const size_t xlen = rd16(h + 10);
    if (off + 12 + xlen > n) return 0;
    size_t x = 0, bsize = 0;
    while (x + 4 <= xlen) {
        const uint8_t *e = h + 12 + x;
        const size_t slen = rd16(e + 2);
        if (e[0] == 'B' && e[1] == 'C' && slen == 2) bsize = (size_t) rd16(e + 4) + 1;
        x += 4 + slen;
    }
    if (!bsize || off + bsize > n) return 0;
    *data_off = 12 + xlen;
    return bsize;
}

bool inflate_block(const uint8_t *src, size_t src_len, uint8_t *dst, size_t dst_len) {
    z_stream zs;
    memset(&zs, 0, sizeof(zs));
    if (inflateInit2(&zs, -15) != Z_OK) return false;
    zs.next_in = (Bytef *) src; zs.avail_in = (uInt) src_len;
    zs.next_out = dst; zs.avail_out = (uInt) dst_len;
    const int rc = inflate(&zs, Z_FINISH);
    const bool ok = (rc == Z_STREAM_END) && zs.total_out == dst_len;
    inflateEnd(&zs);
    return ok;
}

struct Block { size_t coff, data_off, bsize; uint32_t isize; size_t uoff; };

// persistent worker pool (one per reader): spawning 128 threads per parallel loop costs more than a small inflate
struct Pool {
    std::vector<std::thread> workers;
    std::mutex mu;
    std::condition_variable cv_work, cv_done;
    std::function<void(size_t)> fn;
    std::atomic<size_t> next{0};
    size_t n = 0, generation = 0;
    int running = 0;
    bool stop = false;
    explicit Pool(int threads) {
        for (int t = 0; t < threads; t++) workers.emplace_back([this]() { loop(); });
    }
    ~Pool() {
        { std::lock_guard<std::mutex> l(mu); stop = true; }
        cv_work.notify_all();
        for (auto &w : workers) w.join();
    }
    void loop() {
        size_t seen = 0;
        for (;;) {
            {
                std::unique_lock<std::mutex> l(mu);
                cv_work.wait(l, [&]() { return stop || generation != seen; });
                if (stop) return;
                seen = generation;
            }
            for (size_t i; (i = next.fetch_add(1)) < n;) fn(i);
            {
                std::lock_guard<std::mutex> l(mu);
                if (--running == 0) cv_done.notify_all();
            }
        }
    }
    template <typename F> void run(size_t count, F f) {
        if (workers.empty() || count < 2) { for (size_t i = 0; i < count; i++) f(i); return; }
        {
            std::lock_guard<std::mutex> l(mu);
            fn = f; n = count; next = 0; running = (int) workers.size(); generation++;
        }
        cv_work.notify_all();
        for (size_t i; (i = next.fetch_add(1)) < count;) f(i);          // the caller helps
        std::unique_lock<std::mutex> l(mu);
        cv_done.wait(l, [&]() { return running == 0; });
    }
};

struct HostBuf {                 // grow-only; page-locked when a CUDA device is present (faster H2D), plain otherwise
    void *p = nullptr;
    size_t cap = 0;
    bool pinned = false;
    bool reserve(size_t bytes, bool want_pinned) {
        if (bytes <= cap) return true;
        release();
        const size_t want = bytes + bytes / 8 + 256;
        if (want_pinned && cudaMallocHost(&p, want) == cudaSuccess) pinned = true;
        else { cudaGetLastError(); p = malloc(want); pinned = false; }
        if (!p) return false;
        cap = want;
        return true;
    }
    void release() {
        if (p) { if (pinned) cudaFreeHost(p); else free(p); }
        p = nullptr; cap = 0;
    }
    template <typename T> T *as() { return (T *) p; }
};

struct Chunk { uint64_t beg, end; };
// loffset: a CSI bin's lower bound on the virtual offset of any record overlapping the bin (0 in a BAI, which has a linear index)
struct Bin { uint64_t loffset = 0; std::vector<Chunk> chunks; };
struct RefIndex { std::map<uint32_t, Bin> bins; std::vector<uint64_t> linear; };

// The binning scheme of a BAI (min_shift 14, depth 5) or a CSI (SAMv1 5.3): level l (0 = the root) has 8^l bins of 2^shift(l)
// positions, numbered from ((1 << 3l) - 1) / 7.  An index covers [0, 1 << (min_shift + 3 depth)).
struct Binning {
    int min_shift = 14, depth = 5;
    int shift(int l) const { return min_shift + 3 * (depth - l); }
    static uint32_t first(int l) { return (uint32_t) (((1ull << (3 * l)) - 1) / 7); }
    int64_t max_end() const { return 1ll << (min_shift + 3 * depth); }
};

// bins overlapping [beg, end), end <= max_end (SAMv1 5.3 reg2bins)
void reg2bins(const Binning &bn, int64_t beg, int64_t end, std::vector<uint32_t> &out) {
    --end;
    for (int l = 0; l <= bn.depth; l++) {
        const int s = bn.shift(l);
        for (int64_t k = beg >> s; k <= end >> s; ++k) out.push_back(Binning::first(l) + (uint32_t) k);
    }
}

struct RecRef { size_t off; uint32_t l_seq, n_cigar; const uint8_t *cigar; };   // off: start of the record body in the inflated buffer

}  // namespace

struct pb_bam {
    MappedFile f;
    int n_threads = 1;
    Pool *pool = nullptr;
    bool pinned = false;
    std::string text;
    std::vector<std::string> names;
    std::vector<int64_t> lens;
    std::vector<RefIndex> index;
    Binning binning;                    // (14, 5) for a BAI; a CSI's own
    bool csi = false;
    int64_t last_anchors = 0, last_longest_walk = 0;   // of the last pb_bam_fetch_device
    size_t first_record_voff_block = 0;
    // fetch scratch / outputs
    struct RawBuf {                     // grow-only, never zero-filled; contents preserved up to `keep` bytes on growth
        uint8_t *p = nullptr; size_t cap = 0;
        bool ensure(size_t bytes, size_t keep) {
            if (bytes <= cap) return true;
            const size_t want = bytes + bytes / 4 + 4096;
            uint8_t *q = (uint8_t *) malloc(want);
            if (!q) return false;
            if (p && keep) memcpy(q, p, keep);
            free(p); p = q; cap = want;
            return true;
        }
        ~RawBuf() { free(p); }
    } ubuf;
    HostBuf o_pos, o_seq_off, o_cigar_off, o_flag, o_mapq, o_seq, o_qual, o_cigar;
    int64_t n_compressed = 0, n_inflated = 0;
    // device path (pb_bam_fetch_device)
    int device = -1;
    HostBuf c_host;                     // page-locked staging of the compressed blocks
    pb::DevBuf d_comp, d_blocks, d_status, d_ubuf, d_starts, d_stops, d_counts, d_base, d_rec_off, d_info, d_keep32, d_lseq32, d_ncig32,
        d_keep_off, d_so, d_co, d_scal, d_pos, d_seq_off, d_cigar_off, d_flag, d_mapq, d_seq, d_qual, d_cigar;
    cudaStream_t own_stream = nullptr;
    float dev_ms[3] = {0, 0, 0};        // inflate, chain + parse, scatter
    cudaEvent_t dev_evt[4] = {nullptr, nullptr, nullptr, nullptr};
    // hybrid inflate: a share of the BGZF blocks (runs of HOST_RUN consecutive blocks) is inflated by the host pool while the
    // kernel works on the rest, and lands in the same device buffer through a copy stream
    double host_share = 0.0;
    HostBuf u_host;                     // page-locked staging of the host-inflated runs
    cudaStream_t copy_stream = nullptr;
    cudaEvent_t copy_evt = nullptr;
    int64_t n_host_blocks = 0, n_dev_blocks = 0;
};

// cores this process may really use: scheduler affinity capped by the cgroup CPU quota (a container that shows 128 hardware
// threads may be allowed 16)
static int usable_cores() {
    int n = (int) std::max(1u, std::thread::hardware_concurrency());
    cpu_set_t set;
    CPU_ZERO(&set);
    if (sched_getaffinity(0, sizeof(set), &set) == 0) { const int c = CPU_COUNT(&set); if (c > 0) n = std::min(n, c); }
    if (FILE *f = fopen("/sys/fs/cgroup/cpu.max", "r")) {
        char q[64] = {0}; long long period = 0;
        if (fscanf(f, "%63s %lld", q, &period) == 2 && strcmp(q, "max") != 0 && period > 0) {
            const long long quota = atoll(q);
            if (quota > 0) n = (int) std::max(1ll, std::min<long long>(n, quota / period));
        }
        fclose(f);
    }
    return n;
}
constexpr size_t HOST_RUN = 16;

struct pb_fasta {
    MappedFile f;
    struct Entry { std::string name; int64_t len, off, linebases, linewidth; };
    std::vector<Entry> entries;
    std::map<std::string, int> by_name;
    // bgzip-compressed FASTA: the .fai offsets are uncompressed; gzi[k] = (compressed, uncompressed) offset of BGZF block k,
    // block 0 = (0, 0) included.  A fetch inflates only the blocks it needs, into its own buffer (no shared state), so fetches on
    // one handle may run from several threads; the pool is taken with try_lock and a fetch that finds it busy inflates inline.
    bool bgzf = false;
    std::vector<std::pair<uint64_t, uint64_t>> gzi;
    Pool *pool = nullptr;
    std::mutex pool_mu;
    ~pb_fasta() { delete pool; }
};

namespace {

// inflate the blocks covering compressed offsets [c0, c1_block] (c1_block = offset of the LAST block needed)
int inflate_range(pb_bam *b, size_t c0, size_t c1_block, std::vector<Block> &blocks, size_t base, size_t *utotal_out) {
    blocks.clear();
    size_t off = c0, utotal = 0;
    while (off <= c1_block && off < b->f.n) {
        size_t data_off;
        const size_t bs = bgzf_block_size(b->f.p, b->f.n, off, &data_off);
        if (!bs || bs < data_off + 8) { set_error("corrupt BGZF block at offset %zu", off); return PB_ERR_ARG; }       // header + CRC32 + ISIZE must fit
        const uint32_t isize = rd32(b->f.p + off + bs - 4);
        if (isize > 65536) { set_error("BGZF block at offset %zu claims %u inflated bytes (limit 65536)", off, isize); return PB_ERR_ARG; }
        blocks.push_back({off, data_off, bs, isize, utotal});
        utotal += isize;
        off += bs;
    }
    if (!b->ubuf.ensure(base + utotal + 16, base)) { set_error("out of host memory"); return PB_ERR_ARG; }
    uint8_t *out = b->ubuf.p + base;
    *utotal_out = utotal;
    std::atomic<int> bad(0);
    // the compressed bytes are pread() into a per-thread buffer: faulting the mmap'ed file in from 100+ threads at once
    // serialises on the address-space lock (measured: 1.8 GB/s at 460 MB vs 5 GB/s at 115 MB)
    b->pool->run(blocks.size(), [&](size_t i) {
        static thread_local std::vector<uint8_t> cbuf;
        const Block &k = blocks[i];
        if (!k.isize) return;
        if (cbuf.size() < k.bsize) cbuf.resize(65536 + 64);
        const ssize_t got = pread(b->f.fd, cbuf.data(), k.bsize, (off_t) k.coff);
        const uint8_t *src = (got == (ssize_t) k.bsize) ? cbuf.data() : b->f.p + k.coff;
        if (!inflate_block(src + k.data_off, k.bsize - k.data_off - 8, out + k.uoff, k.isize)) bad = 1;
    });
    if (bad) { set_error("BGZF inflate failed"); return PB_ERR_ARG; }
    for (auto &k : blocks) { b->n_compressed += (int64_t) k.bsize; b->n_inflated += k.isize; }
    return PB_OK;
}

size_t upos_of(const std::vector<Block> &blocks, uint64_t voff, size_t utotal) {
    const size_t coff = (size_t) (voff >> 16);
    auto it = std::lower_bound(blocks.begin(), blocks.end(), coff, [](const Block &k, size_t c) { return k.coff < c; });
    if (it == blocks.end() || it->coff != coff) return utotal;         // past the last needed block
    return it->uoff + (size_t) (voff & 0xffff);
}

int load_header(pb_bam *b) {
    // the header sits at the start of the file; inflate blocks until it is complete
    std::vector<Block> blocks;
    size_t want_blocks = 1;
    for (;;) {
        size_t off = 0, last = 0, cnt = 0;
        while (off < b->f.n && cnt < want_blocks) { size_t d; const size_t bs = bgzf_block_size(b->f.p, b->f.n, off, &d); if (!bs) break; last = off; off += bs; cnt++; }
        if (!cnt) { set_error("not a BGZF file"); return PB_ERR_ARG; }
        size_t n = 0;
        PB_TRY(inflate_range(b, 0, last, blocks, 0, &n));
        struct { uint8_t *p; uint8_t *data() const { return p; } } u{b->ubuf.p};
        bool complete = false;
        if (n >= 12 && !memcmp(u.data(), "BAM\1", 4)) {
            const size_t l_text = rd32(u.data() + 4);
            size_t p = 8 + l_text;
            if (p + 4 <= n) {
                const uint32_t n_ref = rd32(u.data() + p);
                p += 4;
                complete = true;
                b->names.clear(); b->lens.clear();
                for (uint32_t i = 0; i < n_ref; i++) {
                    if (p + 4 > n) { complete = false; break; }
                    const uint32_t l_name = rd32(u.data() + p);
                    if (p + 4 + l_name + 4 > n) { complete = false; break; }
                    b->names.emplace_back((const char *) u.data() + p + 4, l_name ? l_name - 1 : 0);
                    b->lens.push_back(rd32(u.data() + p + 4 + l_name));
                    p += 8 + l_name;
                }
                if (complete) b->text.assign((const char *) u.data() + 8, l_text);
            }
        } else if (n >= 4) { set_error("not a BAM file (bad magic)"); return PB_ERR_ARG; }
        if (complete) break;
        if (cnt < want_blocks) { set_error("truncated BAM header"); return PB_ERR_ARG; }
        want_blocks *= 2;
    }
    b->n_compressed = b->n_inflated = 0;
    return PB_OK;
}

int load_bai(pb_bam *b, const char *path) {
    MappedFile f;
    if (!f.open(path)) { set_error("cannot open BAM index %s", path); return PB_ERR_ARG; }
    const uint8_t *p = f.p;
    const size_t n = f.n;
    size_t o = 8;
    if (n < 8 || memcmp(p, "BAI\1", 4)) { f.close(); set_error("%s is not a BAI index", path); return PB_ERR_ARG; }
    const uint32_t n_ref = rd32(p + 4);
    b->index.assign(n_ref, RefIndex());
    for (uint32_t r = 0; r < n_ref; r++) {
        if (o + 4 > n) goto bad;
        {
            const uint32_t n_bin = rd32(p + o); o += 4;
            for (uint32_t i = 0; i < n_bin; i++) {
                if (o + 8 > n) goto bad;
                const uint32_t bin = rd32(p + o), n_chunk = rd32(p + o + 4);
                o += 8;
                if (o + 16ull * n_chunk > n) goto bad;
                auto &v = b->index[r].bins[bin].chunks;
                for (uint32_t c = 0; c < n_chunk; c++, o += 16) v.push_back({rd64(p + o), rd64(p + o + 8)});
            }
            if (o + 4 > n) goto bad;
            const uint32_t n_intv = rd32(p + o); o += 4;
            if (o + 8ull * n_intv > n) goto bad;
            b->index[r].linear.resize(n_intv);
            for (uint32_t i = 0; i < n_intv; i++, o += 8) b->index[r].linear[i] = rd64(p + o);
        }
    }
    f.close();
    return PB_OK;
bad:
    f.close();
    set_error("truncated BAI index %s", path);
    return PB_ERR_ARG;
}

// CSI (the CSIv1 specification): a BGZF file whose payload is magic "CSI\1", min_shift, depth, l_aux, aux, n_ref, then per
// reference n_bin and per bin (bin u32, loffset u64, n_chunk, chunks), optionally n_no_coor u64.  No linear index.
int load_csi(pb_bam *b, const char *path) {
    MappedFile f;
    if (!f.open(path)) { set_error("cannot open BAM index %s", path); return PB_ERR_ARG; }
    std::vector<uint8_t> u;
    for (size_t off = 0; off < f.n;) {
        size_t data_off;
        const size_t bs = bgzf_block_size(f.p, f.n, off, &data_off);
        if (!bs || bs < data_off + 8) { f.close(); set_error("%s is not a BGZF-compressed CSI index (bad block at offset %zu)", path, off); return PB_ERR_ARG; }
        const uint32_t isize = rd32(f.p + off + bs - 4);
        if (isize > 65536) { f.close(); set_error("CSI index %s: block at offset %zu claims %u bytes", path, off, isize); return PB_ERR_ARG; }
        const size_t at = u.size();
        u.resize(at + isize);
        if (isize && !inflate_block(f.p + off + data_off, bs - data_off - 8, u.data() + at, isize)) { f.close(); set_error("CSI index %s: inflate failed", path); return PB_ERR_ARG; }
        off += bs;
    }
    f.close();
    const uint8_t *p = u.data();
    const size_t n = u.size();
    if (n < 16 || memcmp(p, "CSI\1", 4)) { set_error("%s is not a CSI index", path); return PB_ERR_ARG; }
    const int32_t min_shift = rdi32(p + 4), depth = rdi32(p + 8), l_aux = rdi32(p + 12);
    // positions are int32 in a BAM record: a reach past 2^32 would only overflow the bin arithmetic
    if (min_shift < 0 || depth < 0 || min_shift + 3 * depth > 32 || depth > 9) { set_error("CSI index %s: unsupported min_shift %d / depth %d", path, min_shift, depth); return PB_ERR_ARG; }
    if (l_aux < 0 || 16ull + (uint64_t) l_aux + 4 > n) { set_error("truncated CSI index %s", path); return PB_ERR_ARG; }
    size_t o = 16 + (size_t) l_aux;
    const int32_t n_ref = rdi32(p + o); o += 4;
    if (n_ref < 0) { set_error("CSI index %s: negative n_ref", path); return PB_ERR_ARG; }
    b->binning.min_shift = min_shift; b->binning.depth = depth;
    b->index.assign((size_t) n_ref, RefIndex());
    for (int32_t r = 0; r < n_ref; r++) {
        if (o + 4 > n) goto bad;
        {
            const int32_t n_bin = rdi32(p + o); o += 4;
            if (n_bin < 0) goto bad;
            for (int32_t i = 0; i < n_bin; i++) {
                if (o + 16 > n) goto bad;
                const uint32_t bin = rd32(p + o);
                const uint64_t loffset = rd64(p + o + 4);
                const int32_t n_chunk = rdi32(p + o + 12);
                o += 16;
                if (n_chunk < 0 || o + 16ull * (uint64_t) n_chunk > n) goto bad;
                Bin &v = b->index[r].bins[bin];
                v.loffset = loffset;
                for (int32_t c = 0; c < n_chunk; c++, o += 16) v.chunks.push_back({rd64(p + o), rd64(p + o + 8)});
            }
        }
    }
    if (o != n && o + 8 != n) goto bad;                          // nothing but the optional n_no_coor may follow
    b->csi = true;
    return PB_OK;
bad:
    set_error("truncated CSI index %s", path);
    return PB_ERR_ARG;
}

// The index of `path`, the first that exists of <bam>.csi, <name>.csi, <bam>.bai, <name>.bai (name = path without ".bam").
// We believe this is htslib's order (CSI first, each extension appended and then substituted); htslib is not available here to
// confirm it.  A file with both indexes gives the same records through either.
int load_index(pb_bam *b, const char *path) {
    const std::string full(path);
    std::vector<std::string> stems{full};
    if (full.size() > 4 && full.substr(full.size() - 4) == ".bam") stems.push_back(full.substr(0, full.size() - 4));
    struct stat st;
    for (const char *ext : {".csi", ".bai"})
        for (const std::string &s : stems)
            if (stat((s + ext).c_str(), &st) == 0) return ext[1] == 'c' ? load_csi(b, (s + ext).c_str()) : load_bai(b, (s + ext).c_str());
    set_error("cannot open BAM index %s.bai or %s.csi (the BAM file must be indexed)", path, path);
    return PB_ERR_ARG;
}

// The chunks of (tid, [beg, end)) from the bin index, sorted and merged (SAMv1 5.1.1), and the virtual offsets known to start a
// record inside them (`anchors`, optional): the one place pb_bam_fetch and pb_bam_fetch_device turn a query into file spans.
// Chunks ending at or before min_off are dropped: for a BAI min_off is the linear index at beg's 16 kb window; for a CSI it is the
// loffset of the deepest bin on the path from beg's leaf bin up to the root that the index holds (hts_itr_query).  Either is only
// a shortcut: the same records come back without it.  Anchors: the linear index of every window the query touches (BAI) or the
// loffset of every bin it touches (CSI); the device walk starts a thread at each.
void select_chunks(const pb_bam *b, const RefIndex &ri, int64_t beg, int64_t end, std::vector<Chunk> &merged, std::vector<uint64_t> *anchors) {
    const Binning &bn = b->binning;
    std::vector<uint32_t> bins;
    reg2bins(bn, beg, end, bins);
    uint64_t min_off = 0;
    if (!ri.linear.empty()) {
        const size_t w = (size_t) (beg >> 14);
        min_off = ri.linear[std::min(w, ri.linear.size() - 1)];
        if (w >= ri.linear.size()) min_off = ri.linear.back();
    } else if (b->csi) {
        for (int l = bn.depth; l >= 0; l--) {
            auto it = ri.bins.find(Binning::first(l) + (uint32_t) (beg >> bn.shift(l)));
            if (it != ri.bins.end()) { min_off = it->second.loffset; break; }
        }
    }
    std::vector<Chunk> chunks;
    for (uint32_t bin : bins) {
        auto it = ri.bins.find(bin);
        if (it == ri.bins.end()) continue;
        for (const Chunk &c : it->second.chunks) if (c.end > min_off) chunks.push_back(c);
        if (anchors && b->csi) anchors->push_back(it->second.loffset);
    }
    std::sort(chunks.begin(), chunks.end(), [](const Chunk &a, const Chunk &c) { return a.beg < c.beg; });
    merged.clear();
    for (const Chunk &c : chunks) {
        if (!merged.empty() && c.beg <= merged.back().end) merged.back().end = std::max(merged.back().end, c.end);
        else merged.push_back(c);
    }
    if (anchors && !ri.linear.empty()) {
        const size_t w0 = (size_t) (beg >> 14), w1 = std::min((size_t) ((end - 1) >> 14), ri.linear.size() - 1);
        for (size_t w = w0; w <= w1 && w < ri.linear.size(); w++) anchors->push_back(ri.linear[w]);
    }
}

}  // namespace

extern "C" int pb_bam_open(pb_bam_t **out, const char *path, int n_threads) {
    if (!out || !path) { set_error("null argument"); return PB_ERR_ARG; }
    auto *b = new pb_bam();
    if (!b->f.open(path)) { delete b; set_error("cannot open BAM file %s", path); return PB_ERR_ARG; }
    b->n_threads = n_threads > 0 ? n_threads : usable_cores();
    b->pool = new Pool(b->n_threads - 1);
    // share of the blocks left to the host pool in pb_bam_fetch_device: off by default (measured on the chr20-scale files leg: a
    // third of the blocks on 16 cores = 846 ms per step against 862 ms — the fetch thread's pread -> zlib chain takes what the kernel
    // saves); PB_INFLATE_HOST_SHARE or pb_bam_set_host_share turn it on
    b->host_share = 0.0;
    if (const char *e = getenv("PB_INFLATE_HOST_SHARE")) b->host_share = std::min(1.0, std::max(0.0, atof(e)));
    int ndev = 0;
    b->pinned = cudaGetDeviceCount(&ndev) == cudaSuccess && ndev > 0;
    if (!b->pinned) cudaGetLastError();
    int rc = load_header(b);
    if (rc == PB_OK) rc = load_index(b, path);
    if (rc != PB_OK) { b->f.close(); delete b->pool; delete b; return rc; }
    *out = b;
    return PB_OK;
}

extern "C" int pb_bam_close(pb_bam_t *b) {
    if (!b) return PB_OK;
    HostBuf *bufs[] = {&b->o_pos, &b->o_seq_off, &b->o_cigar_off, &b->o_flag, &b->o_mapq, &b->o_seq, &b->o_qual, &b->o_cigar};
    for (auto *x : bufs) x->release();
    b->c_host.release();
    b->u_host.release();
    if (b->copy_stream) cudaStreamDestroy(b->copy_stream);
    if (b->copy_evt) cudaEventDestroy(b->copy_evt);
    pb::DevBuf *dbufs[] = {&b->d_comp, &b->d_blocks, &b->d_status, &b->d_ubuf, &b->d_starts, &b->d_stops, &b->d_counts, &b->d_base, &b->d_rec_off, &b->d_info,
                           &b->d_keep32, &b->d_lseq32, &b->d_ncig32, &b->d_keep_off, &b->d_so, &b->d_co, &b->d_scal, &b->d_pos, &b->d_seq_off, &b->d_cigar_off,
                           &b->d_flag, &b->d_mapq, &b->d_seq, &b->d_qual, &b->d_cigar};
    if (b->device >= 0) { cudaSetDevice(b->device); for (auto *x : dbufs) x->release(); for (auto &e : b->dev_evt) if (e) cudaEventDestroy(e); if (b->own_stream) cudaStreamDestroy(b->own_stream); }
    b->f.close();
    delete b->pool;
    delete b;
    return PB_OK;
}

extern "C" int pb_bam_n_contigs(pb_bam_t *b) { return b ? (int) b->names.size() : 0; }
extern "C" const char *pb_bam_contig_name(pb_bam_t *b, int tid) { return (b && tid >= 0 && tid < (int) b->names.size()) ? b->names[tid].c_str() : nullptr; }
extern "C" int64_t pb_bam_contig_length(pb_bam_t *b, int tid) { return (b && tid >= 0 && tid < (int) b->lens.size()) ? b->lens[tid] : -1; }
extern "C" int pb_bam_contig_id(pb_bam_t *b, const char *name) {
    if (!b || !name) return -1;
    for (size_t i = 0; i < b->names.size(); i++) if (b->names[i] == name) return (int) i;
    return -1;
}
extern "C" const char *pb_bam_header_text(pb_bam_t *b, int64_t *len) {
    if (!b) return nullptr;
    if (len) *len = (int64_t) b->text.size();
    return b->text.c_str();
}
extern "C" int pb_bam_io_stats(pb_bam_t *b, int64_t *compressed, int64_t *inflated) {
    if (!b) return PB_ERR_ARG;
    if (compressed) *compressed = b->n_compressed;
    if (inflated) *inflated = b->n_inflated;
    return PB_OK;
}
// the index's reach: a fetch sees no record at or past it (2^29 for a BAI, 2^(min_shift + 3 depth) for a CSI); -1 on a null handle
extern "C" int64_t pb_bam_index_max_end(pb_bam_t *b) { return b ? b->binning.max_end() : -1; }
// the index format (1 = CSI, 0 = BAI) and its binning
extern "C" int pb_bam_index_info(pb_bam_t *b, int *is_csi, int *min_shift, int *depth) {
    if (!b) return PB_ERR_ARG;
    if (is_csi) *is_csi = b->csi ? 1 : 0;
    if (min_shift) *min_shift = b->binning.min_shift;
    if (depth) *depth = b->binning.depth;
    return PB_OK;
}
// record-start anchors of the last pb_bam_fetch_device (one walking thread each) and the most records one of them walked
extern "C" int pb_bam_fetch_device_anchors(pb_bam_t *b, int64_t *anchors, int64_t *longest_walk) {
    if (!b) return PB_ERR_ARG;
    if (anchors) *anchors = b->last_anchors;
    if (longest_walk) *longest_walk = b->last_longest_walk;
    return PB_OK;
}

extern "C" int pb_bam_fetch(pb_bam_t *b, int tid, int64_t beg, int64_t end, pb_records_t *view) {
    if (!b || !view) { set_error("null argument"); return PB_ERR_ARG; }
    memset(view, 0, sizeof(*view));
    if (tid < 0 || tid >= (int) b->names.size()) { set_error("contig id %d out of range", tid); return PB_ERR_ARG; }
    if (beg < 0) beg = 0;
    if (end > b->binning.max_end()) end = b->binning.max_end();            // the index's reach, as htslib clamps (2^29 for a BAI)
    static const bool dbg = getenv("PB_BAM_DEBUG") != nullptr;
    auto tnow = []() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
    const double t_start = tnow();
    double t_inflate = 0, t_walk = 0;
    int n_groups = 0;
    std::vector<RecRef> recs;
    std::vector<int64_t> rpos;
    std::vector<Block> blocks;
    if (end > beg && tid < (int) b->index.size()) {
        std::vector<Chunk> merged;
        select_chunks(b, b->index[tid], beg, end, merged, nullptr);
        if (!merged.empty()) {
            // one inflate pass over the whole span of the merged chunks would decompress gaps too; inflate per chunk group:
            // chunks whose block ranges touch are handled together
            size_t gi = 0;
            // every group's inflated bytes are appended to b->ubuf; records are remembered as offsets (the buffer may move when it grows)
            size_t store_size = 0;
            std::vector<size_t> rec_store_off;
            bool done = false;
            while (gi < merged.size() && !done) {
                size_t gj = gi;
                uint64_t gend = merged[gi].end;
                while (gj + 1 < merged.size() && (merged[gj + 1].beg >> 16) <= (gend >> 16)) { gj++; gend = std::max(gend, merged[gj].end); }
                const size_t c0 = (size_t) (merged[gi].beg >> 16);
                size_t c1 = (size_t) (gend >> 16);
                if ((gend & 0xffff) == 0 && c1 > c0) c1 -= 1;             // the block at gend is not needed; c1 then points inside the previous block: fine for `off <= c1`
                const double t_a = tnow();
                const size_t base = store_size;
                size_t utotal = 0;
                PB_TRY(inflate_range(b, c0, c1, blocks, base, &utotal));
                const double t_b = tnow();
                t_inflate += t_b - t_a; n_groups++;
                store_size = base + utotal;
                struct { uint8_t *p; uint8_t *data() const { return p; } } u{b->ubuf.p + base};
                // pass 1 (sequential, cheap): hop over the records of the group's chunks, remember those of this contig left of `end`
                std::vector<size_t> cand;
                for (size_t ci = gi; ci <= gj && !done; ci++) {
                    size_t p = upos_of(blocks, merged[ci].beg, utotal);
                    const size_t pe = std::min(upos_of(blocks, merged[ci].end, utotal), utotal);
                    while (p + 4 <= pe) {
                        const uint32_t bs = rd32(u.data() + p);
                        if (bs < 32 || p + 4 + (size_t) bs > utotal) { set_error("BAM record runs past its chunk"); return PB_ERR_ARG; }
                        const uint8_t *r = u.data() + p + 4;
                        // fixed fields + name + cigar + sequence + qualities must fit in the record (a corrupt record would otherwise be
                        // read out of bounds by the parse / scatter passes)
                        if (32ull + r[8] + 4ull * rd16(r + 12) + ((uint64_t) rd32(r + 16) + 1) / 2 + rd32(r + 16) > bs) {
                            set_error("malformed BAM record at inflated offset %zu", p); return PB_ERR_ARG;
                        }
                        const int32_t rtid = rdi32(r), pos = rdi32(r + 4);
                        if (rtid != tid || pos >= end) { if (rtid > tid || (rtid == tid && pos >= end)) { done = true; break; } p += 4 + bs; continue; }
                        cand.push_back(p);
                        p += 4 + bs;
                    }
                }
                // pass 2 (parallel): long-CIGAR convention, reference length, overlap test
                struct Parsed { uint32_t n_cigar; size_t cigar_off; uint8_t keep; };
                std::vector<Parsed> parsed(cand.size());
                const size_t pgrain = 256;
                b->pool->run((cand.size() + pgrain - 1) / pgrain, [&](size_t g) {
                    for (size_t ii = g * pgrain; ii < std::min(cand.size(), (g + 1) * pgrain); ii++) {
                        const size_t p = cand[ii];
                        const uint32_t bs = rd32(u.data() + p);
                        const uint8_t *r = u.data() + p + 4;
                        const int32_t pos = rdi32(r + 4);
                        const uint32_t l_name = r[8], n_cig = rd16(r + 12), l_seq = rd32(r + 16);
                        const uint8_t *cig = r + 32 + l_name;
                        uint32_t n_cigar = n_cig;
                        const uint8_t *cigar = cig;
                        // long CIGAR convention (SAMv1 4.2.2): "<l_seq>S<rlen>N" + CG:B,I tag
                        if (n_cig == 2 && (rd32(cig) & 15) == 4 && (rd32(cig) >> 4) == l_seq && (rd32(cig + 4) & 15) == 3) {
                            const uint8_t *a = cig + 8 + (l_seq + 1) / 2 + l_seq, *ae = r + bs;
                            while (a + 3 <= ae) {
                                const char t0 = (char) a[0], t1 = (char) a[1], ty = (char) a[2];
                                a += 3;
                                size_t sz = 0;
                                if (ty == 'A' || ty == 'c' || ty == 'C') sz = 1;
                                else if (ty == 's' || ty == 'S') sz = 2;
                                else if (ty == 'i' || ty == 'I' || ty == 'f') sz = 4;
                                else if (ty == 'Z' || ty == 'H') { while (a + sz < ae && a[sz]) sz++; sz++; }
                                else if (ty == 'B') {
                                    if (a + 5 > ae) break;
                                    const char st = (char) a[0];
                                    const uint32_t cnt = rd32(a + 1);
                                    const size_t es = (st == 'c' || st == 'C') ? 1 : (st == 's' || st == 'S') ? 2 : 4;
                                    if (t0 == 'C' && t1 == 'G' && st == 'I' && a + 5 + 4ull * cnt <= ae) { n_cigar = cnt; cigar = a + 5; }
                                    sz = 5 + es * cnt;
                                } else break;
                                a += sz;
                            }
                        }
                        int64_t rlen = 0;
                        for (uint32_t k = 0; k < n_cigar; k++) {
                            const uint32_t c = rd32(cigar + 4 * k);
                            const int op = (int) (c & 15);
                            if (op == 0 || op == 2 || op == 3 || op == 7 || op == 8) rlen += c >> 4;
                        }
                        if (n_cigar == 0) rlen = 1;
                        parsed[ii] = {n_cigar, (size_t) (cigar - u.data()), (uint8_t) ((int64_t) pos + rlen > beg)};
                    }
                });
                // pass 3 (sequential): keep the overlapping ones in file order
                for (size_t ii = 0; ii < cand.size(); ii++) {
                    if (!parsed[ii].keep) continue;
                    const uint8_t *r = u.data() + cand[ii] + 4;
                    recs.push_back({base + cand[ii] + 4, rd32(r + 16), parsed[ii].n_cigar, nullptr});
                    rec_store_off.push_back(base + parsed[ii].cigar_off);
                    rpos.push_back(rdi32(r + 4));
                }
                t_walk += tnow() - t_b;
                gi = gj + 1;
            }
            for (size_t i = 0; i < recs.size(); i++) recs[i].cigar = b->ubuf.p + rec_store_off[i];
        }
    }
    const int64_t n = (int64_t) recs.size();
    std::vector<int64_t> so(n + 1, 0), co(n + 1, 0);
    for (int64_t i = 0; i < n; i++) { so[i + 1] = so[i] + recs[i].l_seq; co[i + 1] = co[i] + recs[i].n_cigar; }
    const int64_t nb = so[n], nc = co[n];
    const bool pin = b->pinned;
    if (!b->o_pos.reserve(sizeof(int64_t) * (n + 1), pin) || !b->o_seq_off.reserve(sizeof(int64_t) * (n + 1), pin) ||
        !b->o_cigar_off.reserve(sizeof(int64_t) * (n + 1), pin) || !b->o_flag.reserve(sizeof(uint16_t) * (n + 1), pin) ||
        !b->o_mapq.reserve(n + 1, pin) || !b->o_seq.reserve((size_t) nb / 2 + 16, pin) || !b->o_qual.reserve((size_t) nb + 16, pin) ||
        !b->o_cigar.reserve(sizeof(uint32_t) * (nc + 4), pin)) { set_error("out of host memory"); return PB_ERR_ARG; }
    memcpy(b->o_seq_off.p, so.data(), sizeof(int64_t) * (n + 1));
    memcpy(b->o_cigar_off.p, co.data(), sizeof(int64_t) * (n + 1));
    int64_t *o_pos = b->o_pos.as<int64_t>();
    uint16_t *o_flag = b->o_flag.as<uint16_t>();
    uint8_t *o_mapq = b->o_mapq.as<uint8_t>(), *o_seq = b->o_seq.as<uint8_t>(), *o_qual = b->o_qual.as<uint8_t>();
    uint32_t *o_cigar = b->o_cigar.as<uint32_t>();
    const uint8_t *u = b->ubuf.p;
    auto seq_of = [&](int64_t i) { const uint8_t *r = u + recs[i].off; return r + 32 + r[8] + 4 * (size_t) rd16(r + 12); };
    auto code_at = [](const uint8_t *s, int64_t k) { return (k & 1) ? (s[k >> 1] & 15) : (s[k >> 1] >> 4); };
    const size_t grain = 64;
    b->pool->run(((size_t) n + grain - 1) / grain, [&](size_t g) {
        for (int64_t i = (int64_t) (g * grain); i < std::min<int64_t>(n, (int64_t) ((g + 1) * grain)); i++) {
            const uint8_t *r = u + recs[i].off;
            o_pos[i] = rpos[i];
            o_mapq[i] = r[9];
            o_flag[i] = rd16(r + 14);
            const int64_t l = recs[i].l_seq;
            memcpy(o_cigar + co[i], recs[i].cigar, 4 * (size_t) recs[i].n_cigar);
            const uint8_t *s = seq_of(i);
            memcpy(o_qual + so[i], s + (l + 1) / 2, (size_t) l);
            // nibble-contiguous packing: the byte shared with the previous record is written by THIS record; a trailing half
            // byte only by the last record
            const int64_t o = so[i];
            if (!(o & 1)) {
                memcpy(o_seq + (o >> 1), s, (size_t) (l >> 1));
            } else if (l > 0) {
                int64_t pv = i - 1;
                while (recs[pv].l_seq == 0) pv--;                      // o odd => some earlier record has bases
                o_seq[o >> 1] = (uint8_t) (code_at(seq_of(pv), recs[pv].l_seq - 1) << 4 | code_at(s, 0));
                for (int64_t B = (o + 1) >> 1; B < (o + l) >> 1; B++) {
                    const int64_t k = 2 * B - o;
                    o_seq[B] = (uint8_t) (code_at(s, k) << 4 | code_at(s, k + 1));
                }
            }
        }
    });
    if (nb & 1) {                                                       // trailing half byte: last record that has bases
        int64_t last = n - 1;
        while (recs[last].l_seq == 0) last--;
        o_seq[nb >> 1] = (uint8_t) (code_at(seq_of(last), recs[last].l_seq - 1) << 4);
    }
    if (dbg) fprintf(stderr, "pb_bam_fetch: %d groups, inflate %.1f ms, walk+copy %.1f ms, total %.1f ms, %lld records\n", n_groups, t_inflate, t_walk,
                     tnow() - t_start, (long long) n);
    view->n_records = n;
    view->pos = o_pos; view->seq_off = b->o_seq_off.as<int64_t>(); view->cigar_off = b->o_cigar_off.as<int64_t>();
    view->flag = o_flag; view->mapq = o_mapq; view->seq = o_seq; view->qual = o_qual; view->cigar = o_cigar;
    return PB_OK;
}


// GPU fetch: same records as pb_bam_fetch (file order, htslib overlap rule), delivered as a pb_records_t whose pointers are DEVICE
// pointers owned by the reader (valid until its next pb_bam_fetch_device), ready for pb_get_reads_plan_device.
extern "C" int pb_bam_fetch_device(pb_bam_t *b, int tid, int64_t beg, int64_t end, int device, pb_records_t *view, void *stream_) {
    using namespace pb::bgzf;
    if (!b || !view) { set_error("null argument"); return PB_ERR_ARG; }
    memset(view, 0, sizeof(*view));
    if (tid < 0 || tid >= (int) b->names.size()) { set_error("contig id %d out of range", tid); return PB_ERR_ARG; }
    PB_CUDA(cudaSetDevice(device));
    if (b->device != device) { b->device = device; }
    // stream == NULL: the reader's own NON-BLOCKING stream, so that a prefetch thread's inflate overlaps the kernels the caller
    // queued on the default stream (this function synchronises its stream before it returns: the records are complete)
    if (!stream_ && !b->own_stream) PB_CUDA(cudaStreamCreateWithFlags(&b->own_stream, cudaStreamNonBlocking));
    cudaStream_t st = stream_ ? (cudaStream_t) stream_ : b->own_stream;
    for (auto &e : b->dev_evt) if (!e) PB_CUDA(cudaEventCreate(&e));
    if (beg < 0) beg = 0;
    if (end > b->binning.max_end()) end = b->binning.max_end();
    b->last_anchors = b->last_longest_walk = 0;
    std::vector<Chunk> merged;
    std::vector<uint64_t> anchors;
    if (end > beg && tid < (int) b->index.size()) select_chunks(b, b->index[tid], beg, end, merged, &anchors);
    // ---- block list of every chunk group (groups = chunks whose block ranges touch), compressed bytes into one pinned buffer
    struct Group { size_t c0, c1_end; size_t first_block, n_blocks; uint64_t vbeg, vend; size_t chunk0, chunk1; };
    std::vector<Group> groups;
    std::vector<Block> blocks;                                  // coff = file offset, uoff = offset in the inflated buffer (all groups)
    std::vector<size_t> block_in_off;                           // offset of the block (header included) in the staging buffer
    size_t ctotal = 0, utotal = 0;
    for (size_t gi = 0; gi < merged.size();) {
        size_t gj = gi;
        uint64_t gend = merged[gi].end;
        while (gj + 1 < merged.size() && (merged[gj + 1].beg >> 16) <= (gend >> 16)) { gj++; gend = std::max(gend, merged[gj].end); }
        const size_t c0 = (size_t) (merged[gi].beg >> 16);
        size_t c1 = (size_t) (gend >> 16);
        if ((gend & 0xffff) == 0 && c1 > c0) c1 -= 1;
        Group G;
        G.c0 = c0; G.first_block = blocks.size(); G.vbeg = merged[gi].beg; G.vend = gend; G.chunk0 = gi; G.chunk1 = gj;
        size_t off = c0;
        while (off <= c1 && off < b->f.n) {
            size_t data_off;
            const size_t bs = bgzf_block_size(b->f.p, b->f.n, off, &data_off);
            if (!bs || bs < data_off + 8) { set_error("corrupt BGZF block at offset %zu", off); return PB_ERR_ARG; }
            const uint32_t isize = rd32(b->f.p + off + bs - 4);
            if (isize > 65536) { set_error("BGZF block at offset %zu claims %u bytes", off, isize); return PB_ERR_ARG; }
            blocks.push_back({off, data_off, bs, isize, utotal});
            block_in_off.push_back(ctotal + (off - c0));
            utotal += isize;
            off += bs;
        }
        G.c1_end = off; G.n_blocks = blocks.size() - G.first_block;
        ctotal += off - c0;
        groups.push_back(G);
        gi = gj + 1;
    }
    const int64_t n_blocks = (int64_t) blocks.size();
    if (n_blocks == 0) {
        PB_TRY(b->d_seq_off.reserve(16)); PB_TRY(b->d_cigar_off.reserve(16));
        PB_CUDA(cudaMemsetAsync(b->d_seq_off.p, 0, 8, st)); PB_CUDA(cudaMemsetAsync(b->d_cigar_off.p, 0, 8, st));
        view->seq_off = b->d_seq_off.as<int64_t>(); view->cigar_off = b->d_cigar_off.as<int64_t>();
        PB_CUDA(cudaStreamSynchronize(st));
        return PB_OK;
    }
    if (!b->c_host.reserve(ctotal + 64, true)) { set_error("out of host memory"); return PB_ERR_ARG; }
    {   // parallel pread of the compressed ranges (1 MB slices)
        struct Slice { size_t file_off, dst_off, len; };
        std::vector<Slice> slices;
        size_t dst = 0;
        for (const Group &G : groups) {
            for (size_t o = G.c0; o < G.c1_end; o += (1u << 20)) slices.push_back({o, dst + (o - G.c0), std::min<size_t>(1u << 20, G.c1_end - o)});
            dst += G.c1_end - G.c0;
        }
        uint8_t *cb = b->c_host.as<uint8_t>();
        b->pool->run(slices.size(), [&](size_t i) {
            const Slice &S = slices[i];
            const ssize_t got = pread(b->f.fd, cb + S.dst_off, S.len, (off_t) S.file_off);
            if (got != (ssize_t) S.len) memcpy(cb + S.dst_off, b->f.p + S.file_off, S.len);
        });
    }
    // ---- known record starts: chunk begins + the anchors of select_chunks (linear-index entries of the windows the query touches
    //      for a BAI, loffsets of the bins it touches for a CSI)
    auto upos = [&](uint64_t voff) -> int64_t {
        const size_t coff = (size_t) (voff >> 16);
        auto it = std::lower_bound(blocks.begin(), blocks.end(), coff, [](const Block &k, size_t c) { return k.coff < c; });
        if (it == blocks.end() || it->coff != coff) return -1;
        if ((voff & 0xffff) > it->isize) return -1;
        return (int64_t) (it->uoff + (size_t) (voff & 0xffff));
    };
    std::vector<int64_t> starts, stops;
    for (const Group &G : groups) {
        const Block &lastb = blocks[G.first_block + G.n_blocks - 1];
        int64_t limit = upos(G.vend);
        if (limit < 0) limit = (int64_t) (lastb.uoff + lastb.isize);              // chunk end beyond the last needed block
        std::vector<int64_t> s;
        for (size_t ci = G.chunk0; ci <= G.chunk1; ci++) { const int64_t u0 = upos(merged[ci].beg); if (u0 >= 0 && u0 < limit) s.push_back(u0); }
        for (const uint64_t v : anchors) {
            if (v < G.vbeg || v >= G.vend) continue;
            const int64_t u0 = upos(v);
            if (u0 >= 0 && u0 < limit) s.push_back(u0);
        }
        std::sort(s.begin(), s.end());
        s.erase(std::unique(s.begin(), s.end()), s.end());
        for (size_t i = 0; i < s.size(); i++) { starts.push_back(s[i]); stops.push_back(i + 1 < s.size() ? s[i + 1] : limit); }
    }
    const int n_starts = (int) starts.size();
    // ---- device: copy, inflate.  Runs of HOST_RUN consecutive blocks alternate between the kernel and the host pool in the
    //      ratio host_share; a host run lands at its place in the inflated device buffer through the copy stream
    const int host_of_16 = (int) (b->host_share * 16.0 + 0.5);
    auto on_host = [&](int64_t i) { return (int) ((i / (int64_t) HOST_RUN) % 16) < host_of_16 && blocks[i].isize > 0; };
    std::vector<BlockDesc> desc;
    std::vector<int64_t> dev_block;                             // index of the block each descriptor stands for
    std::vector<int64_t> host_block;
    std::vector<size_t> host_off;                               // offset of the host block in the staging buffer
    size_t htotal = 0;
    desc.reserve((size_t) n_blocks); dev_block.reserve((size_t) n_blocks);
    for (int64_t i = 0; i < n_blocks; i++) {
        const Block &k = blocks[i];
        b->n_compressed += (int64_t) k.bsize; b->n_inflated += k.isize;
        if (on_host(i)) { host_block.push_back(i); host_off.push_back(htotal); htotal += k.isize; continue; }
        desc.push_back({(int64_t) (block_in_off[i] + k.data_off), (int32_t) (k.bsize - k.data_off - 8), (int32_t) k.isize, (int64_t) k.uoff});
        dev_block.push_back(i);
    }
    const int64_t n_dev = (int64_t) desc.size(), n_host = (int64_t) host_block.size();
    b->n_dev_blocks += n_dev; b->n_host_blocks += n_host;
    PB_CUDA(cudaEventRecord(b->dev_evt[0], st));
    PB_TRY(upload(b->d_comp, b->c_host.p, ctotal + 16, st));
    PB_TRY(b->d_status.reserve(sizeof(int) * (n_blocks + 4)));
    PB_TRY(b->d_ubuf.reserve(utotal + 64));
    PB_TRY(b->d_scal.reserve(sizeof(int64_t) * 8));
    PB_CUDA(cudaMemsetAsync(b->d_scal.p, 0, sizeof(int64_t) * 8, st));
    int64_t *sc = b->d_scal.as<int64_t>();                      // [0] n_rec [1] n_keep [2] n_bases [3] n_cigar [4] err (int)
    int *d_err = reinterpret_cast<int *>(sc + 4);
    if (n_dev > 0) {
        PB_TRY(upload(b->d_blocks, desc.data(), sizeof(BlockDesc) * n_dev, st));
        PB_TRY(launch_inflate(b->d_comp.as<uint8_t>(), b->d_blocks.as<BlockDesc>(), n_dev, b->d_ubuf.as<uint8_t>(), b->d_status.as<int>(), st));
    }
    if (n_host > 0) {                                           // while the kernel runs: zlib on the pool, straight from the staged bytes
        if (!b->u_host.reserve(htotal + 64, true)) { set_error("out of host memory"); return PB_ERR_ARG; }
        if (!b->copy_stream) PB_CUDA(cudaStreamCreateWithFlags(&b->copy_stream, cudaStreamNonBlocking));
        if (!b->copy_evt) PB_CUDA(cudaEventCreateWithFlags(&b->copy_evt, cudaEventDisableTiming));
        const uint8_t *cb = b->c_host.as<uint8_t>();
        uint8_t *ub = b->u_host.as<uint8_t>();
        std::atomic<int> bad(0);
        b->pool->run((size_t) n_host, [&](size_t j) {
            const Block &k = blocks[host_block[j]];
            if (!inflate_block(cb + block_in_off[host_block[j]] + k.data_off, k.bsize - k.data_off - 8, ub + host_off[j], k.isize)) bad = 1;
        });
        if (bad) { cudaStreamSynchronize(st); set_error("BGZF inflate failed"); return PB_ERR_ARG; }
        for (int64_t j = 0; j < n_host;) {                      // one copy per run of blocks adjacent in the inflated buffer
            int64_t e = j + 1;
            size_t len = blocks[host_block[j]].isize;
            while (e < n_host && host_block[e] == host_block[e - 1] + 1 &&
                   blocks[host_block[e]].uoff == blocks[host_block[e - 1]].uoff + blocks[host_block[e - 1]].isize) { len += blocks[host_block[e]].isize; e++; }
            PB_CUDA(cudaMemcpyAsync(b->d_ubuf.as<uint8_t>() + blocks[host_block[j]].uoff, ub + host_off[j], len, cudaMemcpyHostToDevice, b->copy_stream));
            j = e;
        }
        PB_CUDA(cudaEventRecord(b->copy_evt, b->copy_stream));
        PB_CUDA(cudaStreamWaitEvent(st, b->copy_evt, 0));
    }
    PB_CUDA(cudaEventRecord(b->dev_evt[1], st));
    // ---- record chains
    int64_t n_rec = 0;
    if (n_starts > 0) {
        PB_TRY(upload(b->d_starts, starts.data(), sizeof(int64_t) * n_starts, st));
        PB_TRY(upload(b->d_stops, stops.data(), sizeof(int64_t) * n_starts, st));
        PB_TRY(b->d_counts.reserve(sizeof(int32_t) * (n_starts + 1)));
        PB_TRY(b->d_base.reserve(sizeof(int64_t) * (n_starts + 2)));
        k_chain<0><<<(unsigned) ceil_div(n_starts, 128), 128, 0, st>>>(b->d_ubuf.as<uint8_t>(), b->d_starts.as<int64_t>(), b->d_stops.as<int64_t>(), n_starts,
                                                                       b->d_counts.as<int32_t>(), nullptr, nullptr, d_err);
        k_scan_excl<<<1, 1024, 0, st>>>(b->d_counts.as<int32_t>(), b->d_base.as<int64_t>(), n_starts, sc + 0);
    }
    std::vector<int> h_status((size_t) n_dev + 1);
    std::vector<int32_t> h_counts((size_t) n_starts + 1, 0);      // records walked from each anchor (reported, not used)
    int64_t h_sc[5] = {0, 0, 0, 0, 0};
    if (n_dev > 0) PB_CUDA(cudaMemcpyAsync(h_status.data(), b->d_status.p, sizeof(int) * n_dev, cudaMemcpyDeviceToHost, st));
    if (n_starts > 0) PB_CUDA(cudaMemcpyAsync(h_counts.data(), b->d_counts.p, sizeof(int32_t) * n_starts, cudaMemcpyDeviceToHost, st));
    PB_CUDA(cudaMemcpyAsync(h_sc, sc, sizeof(h_sc), cudaMemcpyDeviceToHost, st));
    PB_CUDA(cudaStreamSynchronize(st));
    b->last_anchors = n_starts;
    b->last_longest_walk = n_starts > 0 ? *std::max_element(h_counts.begin(), h_counts.begin() + n_starts) : 0;
    for (int64_t i = 0; i < n_dev; i++)
        if (h_status[i]) { set_error("BGZF inflate failed on the GPU: block at file offset %zu, status %d", blocks[dev_block[i]].coff, h_status[i]); return PB_ERR_ARG; }
    if ((int) h_sc[4]) { set_error("BAM record chain is inconsistent with the index (code %d)", (int) h_sc[4]); return PB_ERR_ARG; }
    n_rec = h_sc[0];
    int64_t n_keep = 0, nb = 0, nc = 0;
    if (n_rec > 0) {
        PB_TRY(b->d_rec_off.reserve(sizeof(int64_t) * n_rec));
        PB_TRY(b->d_info.reserve(sizeof(RecInfo) * n_rec));
        PB_TRY(b->d_keep32.reserve(sizeof(int32_t) * n_rec)); PB_TRY(b->d_lseq32.reserve(sizeof(int32_t) * n_rec)); PB_TRY(b->d_ncig32.reserve(sizeof(int32_t) * n_rec));
        PB_TRY(b->d_keep_off.reserve(sizeof(int64_t) * (n_rec + 1))); PB_TRY(b->d_so.reserve(sizeof(int64_t) * (n_rec + 1))); PB_TRY(b->d_co.reserve(sizeof(int64_t) * (n_rec + 1)));
        k_chain<1><<<(unsigned) ceil_div(n_starts, 128), 128, 0, st>>>(b->d_ubuf.as<uint8_t>(), b->d_starts.as<int64_t>(), b->d_stops.as<int64_t>(), n_starts, nullptr,
                                                                       b->d_base.as<int64_t>(), b->d_rec_off.as<int64_t>(), d_err);
        k_rec_parse<<<(unsigned) ceil_div(n_rec, 128), 128, 0, st>>>(b->d_ubuf.as<uint8_t>(), b->d_rec_off.as<int64_t>(), n_rec, tid, beg, end, b->d_info.as<RecInfo>(),
                                                                     b->d_keep32.as<int32_t>(), b->d_lseq32.as<int32_t>(), b->d_ncig32.as<int32_t>(), d_err);
        k_scan_excl<<<1, 1024, 0, st>>>(b->d_keep32.as<int32_t>(), b->d_keep_off.as<int64_t>(), n_rec, sc + 1);
        k_scan_excl<<<1, 1024, 0, st>>>(b->d_lseq32.as<int32_t>(), b->d_so.as<int64_t>(), n_rec, sc + 2);
        k_scan_excl<<<1, 1024, 0, st>>>(b->d_ncig32.as<int32_t>(), b->d_co.as<int64_t>(), n_rec, sc + 3);
        PB_CUDA(cudaMemcpyAsync(h_sc, sc, sizeof(h_sc), cudaMemcpyDeviceToHost, st));
        PB_CUDA(cudaStreamSynchronize(st));
        if ((int) h_sc[4]) { set_error("malformed BAM record (code %d)", (int) h_sc[4]); return PB_ERR_ARG; }
        n_keep = h_sc[1]; nb = h_sc[2]; nc = h_sc[3];
    }
    PB_CUDA(cudaEventRecord(b->dev_evt[2], st));
    PB_TRY(b->d_pos.reserve(sizeof(int64_t) * (n_keep + 1))); PB_TRY(b->d_seq_off.reserve(sizeof(int64_t) * (n_keep + 2)));
    PB_TRY(b->d_cigar_off.reserve(sizeof(int64_t) * (n_keep + 2))); PB_TRY(b->d_flag.reserve(sizeof(uint16_t) * (n_keep + 1)));
    PB_TRY(b->d_mapq.reserve(n_keep + 1)); PB_TRY(b->d_seq.reserve((size_t) nb / 2 + 16)); PB_TRY(b->d_qual.reserve((size_t) nb + 16));
    PB_TRY(b->d_cigar.reserve(sizeof(uint32_t) * (nc + 4)));
    if (n_rec > 0 && n_keep > 0) {
        k_rec_scatter<<<(unsigned) ceil_div(n_rec * 32, 256), 256, 0, st>>>(b->d_ubuf.as<uint8_t>(), b->d_rec_off.as<int64_t>(), b->d_info.as<RecInfo>(),
                                                                           b->d_keep_off.as<int64_t>(), b->d_so.as<int64_t>(), b->d_co.as<int64_t>(), n_rec,
                                                                           b->d_pos.as<int64_t>(), b->d_seq_off.as<int64_t>(), b->d_cigar_off.as<int64_t>(),
                                                                           b->d_flag.as<uint16_t>(), b->d_mapq.as<uint8_t>(), b->d_seq.as<uint8_t>(),
                                                                           b->d_qual.as<uint8_t>(), b->d_cigar.as<uint32_t>());
        k_rec_tail<<<1, 32, 0, st>>>(b->d_ubuf.as<uint8_t>(), b->d_rec_off.as<int64_t>(), b->d_info.as<RecInfo>(), n_rec, nb, b->d_seq.as<uint8_t>());
    }
    // closing offsets seq_off[n_keep] = nb, cigar_off[n_keep] = nc
    const int64_t tails[2] = {nb, nc};
    PB_CUDA(cudaMemcpyAsync(b->d_seq_off.as<int64_t>() + n_keep, &tails[0], sizeof(int64_t), cudaMemcpyHostToDevice, st));
    PB_CUDA(cudaMemcpyAsync(b->d_cigar_off.as<int64_t>() + n_keep, &tails[1], sizeof(int64_t), cudaMemcpyHostToDevice, st));
    PB_CUDA(cudaGetLastError());
    PB_CUDA(cudaEventRecord(b->dev_evt[3], st));
    PB_CUDA(cudaStreamSynchronize(st));
    for (int i = 0; i < 3; i++) cudaEventElapsedTime(&b->dev_ms[i], b->dev_evt[i], b->dev_evt[i + 1]);
    view->n_records = n_keep;
    view->pos = b->d_pos.as<int64_t>(); view->seq_off = b->d_seq_off.as<int64_t>(); view->cigar_off = b->d_cigar_off.as<int64_t>();
    view->flag = b->d_flag.as<uint16_t>(); view->mapq = b->d_mapq.as<uint8_t>(); view->seq = b->d_seq.as<uint8_t>();
    view->qual = b->d_qual.as<uint8_t>(); view->cigar = b->d_cigar.as<uint32_t>();
    return PB_OK;
}

// device time (ms) of the last pb_bam_fetch_device: [H2D + inflate, record chains + parse, scatter]
extern "C" int pb_bam_fetch_device_timings(pb_bam_t *b, float *ms3) {
    if (!b || !ms3) return PB_ERR_ARG;
    for (int i = 0; i < 3; i++) ms3[i] = b->dev_ms[i];
    return PB_OK;
}

// share of the BGZF blocks pb_bam_fetch_device leaves to the host pool (0 = all on the GPU — the default —, 1 = all on the host;
// env PB_INFLATE_HOST_SHARE overrides the default)
extern "C" int pb_bam_set_host_share(pb_bam_t *b, double share) {
    if (!b || !(share >= 0.0 && share <= 1.0)) { set_error("host share must be in [0, 1]"); return PB_ERR_ARG; }
    b->host_share = share;
    return PB_OK;
}
// blocks inflated by the host pool / by the kernel in all pb_bam_fetch_device calls so far
extern "C" int pb_bam_inflate_split(pb_bam_t *b, int64_t *host_blocks, int64_t *device_blocks) {
    if (!b) return PB_ERR_ARG;
    if (host_blocks) *host_blocks = b->n_host_blocks;
    if (device_blocks) *device_blocks = b->n_dev_blocks;
    return PB_OK;
}

// diagnostics / tests: inflate `n_blocks` raw DEFLATE streams on the GPU (h_in_off / h_in_len / h_out_len per stream, outputs
// concatenated in order); h_status[i] != 0 marks a stream the kernel rejected.  spec: 1 / 0 = the speculative / one-decoder
// symbol loop, -1 = whichever launch_inflate picks
static int inflate_blocks_host(const uint8_t *h_comp, int64_t comp_bytes, const int64_t *h_in_off, const int32_t *h_in_len, const int32_t *h_out_len,
                               int64_t n_blocks, uint8_t *h_out, int32_t *h_status, void *stream_, int spec) {
    using namespace pb::bgzf;
    if (!h_comp || !h_in_off || !h_in_len || !h_out_len || !h_out || !h_status) { set_error("null argument"); return PB_ERR_ARG; }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev < 1) { set_error("no CUDA device: libpepper_b200 has no CPU fallback"); return PB_ERR_CUDA; }
    cudaStream_t st = (cudaStream_t) stream_;
    std::vector<BlockDesc> desc((size_t) n_blocks);
    int64_t utotal = 0;
    for (int64_t i = 0; i < n_blocks; i++) {
        if (h_in_off[i] < 0 || h_in_off[i] + h_in_len[i] > comp_bytes || h_out_len[i] < 0) { set_error("stream %lld out of bounds", (long long) i); return PB_ERR_ARG; }
        desc[i] = {h_in_off[i], h_in_len[i], h_out_len[i], utotal};
        utotal += h_out_len[i];
    }
    DevBuf dc, db, ds, du;
    int rc = PB_OK;
    do {
        if ((rc = upload(dc, h_comp, (size_t) comp_bytes, st)) != PB_OK) break;
        if ((rc = upload(db, desc.data(), sizeof(BlockDesc) * n_blocks, st)) != PB_OK) break;
        if ((rc = ds.reserve(sizeof(int) * (n_blocks + 1))) != PB_OK) break;
        if ((rc = du.reserve((size_t) utotal + 64)) != PB_OK) break;
        if (n_blocks && spec < 0 && (rc = launch_inflate(dc.as<uint8_t>(), db.as<BlockDesc>(), n_blocks, du.as<uint8_t>(), ds.as<int>(), st)) != PB_OK) break;
        if (n_blocks && spec >= 0) {
            const unsigned grid = (unsigned) ceil_div(n_blocks, WARPS_PER_CTA);
            if (spec) k_bgzf_inflate<true><<<grid, 32 * WARPS_PER_CTA, 0, st>>>(dc.as<uint8_t>(), db.as<BlockDesc>(), (int) n_blocks, du.as<uint8_t>(), ds.as<int>());
            else k_bgzf_inflate<false><<<grid, 32 * WARPS_PER_CTA, 0, st>>>(dc.as<uint8_t>(), db.as<BlockDesc>(), (int) n_blocks, du.as<uint8_t>(), ds.as<int>());
            if (cudaGetLastError() != cudaSuccess) { set_error("inflate launch failed"); rc = PB_ERR_CUDA; break; }
        }
        cudaMemcpyAsync(h_status, ds.p, sizeof(int) * n_blocks, cudaMemcpyDeviceToHost, st);
        if (utotal) cudaMemcpyAsync(h_out, du.p, (size_t) utotal, cudaMemcpyDeviceToHost, st);
        if (cudaStreamSynchronize(st) != cudaSuccess) { set_error("inflate kernel failed: %s", cudaGetErrorString(cudaGetLastError())); rc = PB_ERR_CUDA; }
    } while (0);
    dc.release(); db.release(); ds.release(); du.release();
    return rc;
}
extern "C" int pb_inflate_blocks_host(const uint8_t *h_comp, int64_t comp_bytes, const int64_t *h_in_off, const int32_t *h_in_len, const int32_t *h_out_len,
                                      int64_t n_blocks, uint8_t *h_out, int32_t *h_status, void *stream) {
    return inflate_blocks_host(h_comp, comp_bytes, h_in_off, h_in_len, h_out_len, n_blocks, h_out, h_status, stream, -1);
}
extern "C" int pb_test_inflate_blocks(const uint8_t *h_comp, int64_t comp_bytes, const int64_t *h_in_off, const int32_t *h_in_len, const int32_t *h_out_len,
                                      int64_t n_blocks, uint8_t *h_out, int32_t *h_status, void *stream, int spec) {
    if (spec != 0 && spec != 1) { set_error("pb_test_inflate_blocks: spec must be 0 or 1"); return PB_ERR_ARG; }
    return inflate_blocks_host(h_comp, comp_bytes, h_in_off, h_in_len, h_out_len, n_blocks, h_out, h_status, stream, spec);
}

// ----------------------------------------------------------------------------------------------------------- FASTA
extern "C" int pb_fasta_open(pb_fasta_t **out, const char *path) {
    if (!out || !path) { set_error("null argument"); return PB_ERR_ARG; }
    auto *f = new pb_fasta();
    if (!f->f.open(path)) { delete f; set_error("cannot open FASTA file %s", path); return PB_ERR_ARG; }
    if (f->f.n >= 2 && f->f.p[0] == 0x1f && f->f.p[1] == 0x8b) {
        size_t d;
        if (!bgzf_block_size(f->f.p, f->f.n, 0, &d)) { f->f.close(); delete f; set_error("%s is compressed with gzip, not bgzip: it cannot be indexed for random access", path); return PB_ERR_ARG; }
        const std::string gzi = std::string(path) + ".gzi";
        MappedFile g;
        if (!g.open(gzi.c_str())) { f->f.close(); delete f; set_error("cannot open %s: a bgzip-compressed FASTA needs its .gzi index", gzi.c_str()); return PB_ERR_ARG; }
        const uint64_t n_entries = g.n >= 8 ? rd64(g.p) : 0;
        if (g.n < 8 || g.n != 8 + 16 * n_entries) { g.close(); f->f.close(); delete f; set_error("malformed .gzi index %s", gzi.c_str()); return PB_ERR_ARG; }
        f->gzi.emplace_back(0, 0);
        for (uint64_t i = 0; i < n_entries; i++) f->gzi.emplace_back(rd64(g.p + 8 + 16 * i), rd64(g.p + 16 + 16 * i));
        g.close();
        for (size_t i = 1; i < f->gzi.size(); i++)
            if (f->gzi[i].first <= f->gzi[i - 1].first || f->gzi[i].second < f->gzi[i - 1].second || f->gzi[i].first >= f->f.n) {
                f->f.close(); delete f; set_error("malformed .gzi index %s: offsets out of order or past the file", gzi.c_str()); return PB_ERR_ARG;
            }
        f->bgzf = true;
        f->pool = new Pool(std::min(8, usable_cores()) - 1);
    }
    MappedFile idx;
    const std::string fai = std::string(path) + ".fai";
    if (!idx.open(fai.c_str())) { f->f.close(); delete f; set_error("cannot open FASTA index %s (file must be indexed)", fai.c_str()); return PB_ERR_ARG; }
    const char *p = (const char *) idx.p, *e = p + idx.n;
    while (p < e) {
        const char *nl = (const char *) memchr(p, '\n', (size_t) (e - p));
        const char *le = nl ? nl : e;
        std::string line(p, le);
        p = nl ? nl + 1 : e;
        if (line.empty()) continue;
        pb_fasta::Entry en;
        size_t t0 = line.find('\t');
        if (t0 == std::string::npos) continue;
        en.name = line.substr(0, t0);
        long long v[4] = {0, 0, 0, 0};
        if (sscanf(line.c_str() + t0 + 1, "%lld\t%lld\t%lld\t%lld", &v[0], &v[1], &v[2], &v[3]) != 4) { idx.close(); f->f.close(); delete f; set_error("malformed .fai line"); return PB_ERR_ARG; }
        en.len = v[0]; en.off = v[1]; en.linebases = v[2]; en.linewidth = v[3];
        f->by_name[en.name] = (int) f->entries.size();
        f->entries.push_back(en);
    }
    idx.close();
    *out = f;
    return PB_OK;
}

extern "C" int pb_fasta_close(pb_fasta_t *f) {
    if (!f) return PB_OK;
    f->f.close();
    delete f;
    return PB_OK;
}
extern "C" int pb_fasta_n_contigs(pb_fasta_t *f) { return f ? (int) f->entries.size() : 0; }
extern "C" const char *pb_fasta_contig_name(pb_fasta_t *f, int i) { return (f && i >= 0 && i < (int) f->entries.size()) ? f->entries[i].name.c_str() : nullptr; }
extern "C" int64_t pb_fasta_contig_length(pb_fasta_t *f, const char *name) {
    if (!f || !name) return -1;
    auto it = f->by_name.find(name);
    return it == f->by_name.end() ? -1 : f->entries[it->second].len;
}

// FASTA_handler::get_reference_sequence(region, start, stop) == faidx_fetch_seq(fai, region, start, stop - 1, &len)
// (fasta_handler.cpp:31-50): inclusive end, both ends clamped into the contig like htslib 1.9 faidx.c does, characters
// returned as stored (no case folding).  *len = -2 when the contig is absent (and PB_ERR_ARG is returned).
extern "C" int pb_fasta_fetch(pb_fasta_t *f, const char *name, int64_t start, int64_t stop, char *out, int64_t cap, int64_t *len) {
    if (!f || !name || !len) { set_error("null argument"); return PB_ERR_ARG; }
    auto it = f->by_name.find(name);
    if (it == f->by_name.end()) { *len = -2; set_error("CHROMOSOME NAME NOT PRESENT IN REFERENCE FASTA FILE: %s", name); return PB_ERR_ARG; }
    const pb_fasta::Entry &e = f->entries[it->second];
    int64_t b = start, en = stop - 1;
    if (en < b) b = en;
    if (b < 0) b = 0; else if (e.len <= b) b = e.len - 1;
    if (en < 0) en = 0; else if (e.len <= en) en = e.len - 1;
    const int64_t n = (e.len > 0) ? en - b + 1 : 0;
    *len = n;
    if (n > cap) return PB_ERR_CAPACITY;
    if (!out || n <= 0) return PB_OK;
    // the bytes of [b, en] in the file's line layout are [u0, u1): straight from the mapping, or from the BGZF blocks that hold them
    auto byte_of = [&](int64_t i) { return e.off + (i / e.linebases) * e.linewidth + i % e.linebases; };
    const int64_t u0 = byte_of(b), u1 = byte_of(en) + 1;
    const uint8_t *src = f->f.p;
    size_t src_n = f->f.n;
    int64_t base = 0;
    std::vector<uint8_t> ubuf;
    if (f->bgzf) {
        auto block_of = [&](int64_t u) {
            return (size_t) (std::upper_bound(f->gzi.begin(), f->gzi.end(), (uint64_t) u, [](uint64_t v, const std::pair<uint64_t, uint64_t> &g) { return v < g.second; }) - f->gzi.begin()) - 1;
        };
        const size_t k0 = block_of(u0), k1 = block_of(u1 - 1);
        std::vector<Block> blocks;
        size_t total = 0;
        for (size_t k = k0; k <= k1; k++) {
            size_t data_off;
            const size_t coff = (size_t) f->gzi[k].first;
            const size_t bs = bgzf_block_size(f->f.p, f->f.n, coff, &data_off);
            if (!bs || bs < data_off + 8) { set_error("corrupt BGZF block at offset %zu of the FASTA", coff); return PB_ERR_ARG; }
            const uint32_t isize = rd32(f->f.p + coff + bs - 4);
            const bool next_ok = k + 1 < f->gzi.size() ? (f->gzi[k + 1].first == coff + bs && f->gzi[k + 1].second == f->gzi[k].second + isize) : true;
            if (isize > 65536 || !next_ok) { set_error("the .gzi index does not match the BGZF blocks of the FASTA at offset %zu", coff); return PB_ERR_ARG; }
            blocks.push_back({coff, data_off, bs, isize, total});
            total += isize;
        }
        ubuf.resize(total + 1);
        std::atomic<int> bad(0);
        auto one = [&](size_t i) {
            const Block &k = blocks[i];
            if (k.isize && !inflate_block(f->f.p + k.coff + k.data_off, k.bsize - k.data_off - 8, ubuf.data() + k.uoff, k.isize)) bad = 1;
        };
        std::unique_lock<std::mutex> lk(f->pool_mu, std::try_to_lock);
        if (lk.owns_lock()) f->pool->run(blocks.size(), one);
        else for (size_t i = 0; i < blocks.size(); i++) one(i);
        if (bad) { set_error("BGZF inflate failed in the FASTA"); return PB_ERR_ARG; }
        src = ubuf.data(); src_n = total; base = (int64_t) f->gzi[k0].second;
    }
    int64_t w = 0;
    for (int64_t i = b; i <= en;) {
        const int64_t col = i % e.linebases;
        const int64_t take = std::min(e.linebases - col, en - i + 1);
        const int64_t off = byte_of(i) - base;
        if (off < 0 || (size_t) (off + take) > src_n) { set_error("FASTA index points past the end of the file"); return PB_ERR_ARG; }
        memcpy(out + w, src + off, (size_t) take);
        w += take; i += take;
    }
    return PB_OK;
}
