// block_manager.cpp -- C++ host-side mirror of garage_block::manager::BlockManager for the
// erasure-coded block path (see include/garage_block_manager.h for the mirrored surface and
// the reference file:line of every method).  Host code only: it reaches the GPU exclusively
// through the C ABI in include/garage_ec.h, exactly like the Rust shim of INTEGRATION.md would.
//
// Row f1 (batching front-end): rpc_put_block / reconstructing GETs / resync workers are called
// from many threads (reference: <= 3 blocks in flight per PUT, src/api/s3/put.rs:42; 8 resync
// workers, src/block/resync.rs:43).  One block per GPU call cannot amortise launch + PCIe
// latency, so calls are queued and dispatcher threads hand the GPU whole batches.  Data movement
// on the host is done by the CALLING threads, in parallel: a PUT lands its block in a pinned slot
// and later stores its shards straight out of the dispatcher's pinned parity buffer; a degraded
// GET / a resync worker reads the surviving shards from the node stores straight into its own
// pinned stripe slot, and the batch handed to the GPU is a list of slot pointers
// (garage_ec_reconstruct_stripes).  The dispatchers only issue the batch call.
#include "../../include/garage_block_manager.h"
#include "../../include/garage_ec.h"
#include "../../include/garage_placement.h"

#include <algorithm>
#include <array>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cctype>
#include <cerrno>
#include <climits>
#include <cstddef>
#include <cstdio>
#include <cstring>
#include <deque>
#include <filesystem>
#include <functional>
#include <future>
#include <memory>
#include <mutex>
#include <new>
#include <numeric>
#include <random>
#include <set>
#include <string>
#include <type_traits>
#include <thread>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include <fcntl.h>
#include <sys/mman.h>
#include <sys/random.h>
#include <sys/stat.h>
#include <sys/syscall.h>
#include <unistd.h>

namespace {

using Hash = std::array<uint8_t, 32>;
using Clock = std::chrono::steady_clock;
// the microseconds since t0: what a call adds to its *_us counter
inline uint64_t us_since(Clock::time_point t0)
{
    return (uint64_t)std::chrono::duration_cast<std::chrono::microseconds>(Clock::now() - t0).count();
}
struct HashHasher {
    size_t operator()(const Hash &h) const
    {
        size_t v;
        memcpy(&v, h.data() + 8, sizeof(v));  // content hashes are uniform already
        return v;
    }
};

Hash to_hash(const uint8_t *p)
{
    Hash h;
    memcpy(h.data(), p, 32);
    return h;
}

// copy into a pinned buffer the GPU reads next (landing copy of a PUT, survivors of a degraded GET)
inline void copy_for_dma(uint8_t *dst, const uint8_t *src, size_t n) { garage_ec_copy_for_dma(dst, src, n); }

uint32_t adler32_small(const uint8_t *p, size_t n)
{
    uint32_t a = 1, b = 0;
    for (size_t i = 0; i < n; i++) {
        a = (a + p[i]) % 65521;
        b = (b + a) % 65521;
    }
    return (b << 16) | a;
}

// ---------------------------------------------------------------- one node's local store
// mirrors BlockManagerLocked::write_block_inner / find_block / read_block_from /
// move_block_to_corrupted (src/block/manager.rs:720-819) with a map instead of a directory tree
struct ShardMeta {
    int index = -1;          // which of the k+m shards
    uint32_t block_len = 0;  // unpadded length of the whole block
    uint32_t shard_len = 0;
    uint8_t sum_kind = 0;    // GARAGE_EC_SUM_* of `sum`
    Hash sum{};              // integrity tag of the shard bytes (row f2)
};
// Memory of the in-memory node stores.  A 1 MiB PUT stores k+m = 14 buffers of ~100 KB: through malloc that is
// 1.4 MiB of fresh pages per block (~360 page faults, plus the allocator's own heap growth), all against one
// address space -- at 12 000 blocks/s the process spends its time in the kernel's fault path, not copying.  The arena
// carves cells out of large anonymous regions, hands freed cells back out (LIFO per size class), and can be
// filled ahead of time (reserve), the way the page cache of a disk-backed node is not charged to a PUT either.
class ShardArena {
public:
    static ShardArena &instance()
    {
        static ShardArena *a = new ShardArena();  // never destroyed: shards may outlive any one manager
        return *a;
    }
    static size_t cell_size(size_t n) { return n <= 4096 ? (n + 63) / 64 * 64 : (n + 4095) / 4096 * 4096; }
    uint8_t *alloc(size_t n, size_t *cap)
    {
        const size_t c = cell_size(n);
        *cap = c;
        if (c > kRegion / 4) return static_cast<uint8_t *>(malloc(c));
        std::lock_guard<std::mutex> lk(mu_);
        auto it = free_.find(c);
        if (it != free_.end() && !it->second.empty()) {
            uint8_t *p = it->second.back();
            it->second.pop_back();
            return p;
        }
        return carve(c);
    }
    void free(uint8_t *p, size_t cap)
    {
        if (!p) return;
        if (cap > kRegion / 4) return ::free(p);
        std::lock_guard<std::mutex> lk(mu_);
        free_[cap].push_back(p);
    }
    // make `count` cells for buffers of `n` bytes available with their pages already present
    void reserve(size_t n, size_t count)
    {
        const size_t c = cell_size(n);
        if (c > kRegion / 4 || count == 0) return;
        std::vector<uint8_t *> cells;
        {
            std::lock_guard<std::mutex> lk(mu_);
            auto &fl = free_[c];
            if (fl.size() >= count) return;  // recycled cells have been written before
            count -= fl.size();
            cells.reserve(count);
            for (size_t i = 0; i < count; i++) {
                uint8_t *p = carve(c);
                if (!p) break;
                cells.push_back(p);
            }
        }
        const unsigned hw = std::max(1u, std::thread::hardware_concurrency());
        const size_t nt = std::min<size_t>(std::min(hw, 32u), cells.size() / 64 + 1);
        std::vector<std::thread> th;
        for (size_t t = 0; t < nt; t++)
            th.emplace_back([&, t] {
                for (size_t i = t; i < cells.size(); i += nt)
                    for (size_t o = 0; o < c; o += 4096) reinterpret_cast<volatile uint8_t *>(cells[i])[o] = 0;
            });
        for (auto &x : th) x.join();
        std::lock_guard<std::mutex> lk(mu_);
        auto &fl = free_[c];
        fl.insert(fl.end(), cells.begin(), cells.end());
    }

private:
    static constexpr size_t kRegion = (size_t)256 << 20;
    std::mutex mu_;
    uint8_t *cur_ = nullptr, *end_ = nullptr;
    std::unordered_map<size_t, std::vector<uint8_t *>> free_;
    uint8_t *carve(size_t c)  // mu_ held
    {
        if (cur_ == nullptr || (size_t)(end_ - cur_) < c) {
            void *m = mmap(nullptr, kRegion, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
            if (m == MAP_FAILED) return nullptr;
            cur_ = static_cast<uint8_t *>(m);  // the tail of the previous region is abandoned (< one cell)
            end_ = cur_ + kRegion;
        }
        uint8_t *p = cur_;
        cur_ += c;
        return p;
    }
};

// owning byte buffer in arena memory, with the slice of std::vector's interface the store uses
class ShardBytes {
public:
    ShardBytes() = default;
    ShardBytes(const ShardBytes &o) { assign(o.p_, o.p_ + o.n_); }
    ShardBytes(ShardBytes &&o) noexcept : p_(o.p_), n_(o.n_), cap_(o.cap_) { o.p_ = nullptr, o.n_ = o.cap_ = 0; }
    ShardBytes &operator=(const ShardBytes &o)
    {
        if (this != &o) assign(o.p_, o.p_ + o.n_);
        return *this;
    }
    ShardBytes &operator=(ShardBytes &&o) noexcept
    {
        if (this != &o) {
            ShardArena::instance().free(p_, cap_);
            p_ = o.p_, n_ = o.n_, cap_ = o.cap_;
            o.p_ = nullptr, o.n_ = o.cap_ = 0;
        }
        return *this;
    }
    ~ShardBytes() { ShardArena::instance().free(p_, cap_); }
    void resize(size_t n)  // contents are not preserved across a growth (no caller needs that)
    {
        if (n > cap_) {
            ShardArena::instance().free(p_, cap_);
            p_ = nullptr, cap_ = 0;
            p_ = ShardArena::instance().alloc(n, &cap_);
            if (!p_) {
                n_ = cap_ = 0;
                throw std::bad_alloc();
            }
        }
        n_ = n;
    }
    void assign(const uint8_t *b, const uint8_t *e)
    {
        const size_t n = (size_t)(e - b);
        if (p_ && b >= p_ && b < p_ + cap_) {  // source inside this buffer
            memmove(p_, b, n);
            n_ = n;
            return;
        }
        resize(n);
        if (n) memcpy(p_, b, n);
    }
    uint8_t *data() { return p_; }
    const uint8_t *data() const { return p_; }
    size_t size() const { return n_; }
    bool empty() const { return n_ == 0; }
    uint8_t &operator[](size_t i) { return p_[i]; }

private:
    uint8_t *p_ = nullptr;
    size_t n_ = 0, cap_ = 0;
};

struct StoredShard : ShardMeta {
    ShardBytes bytes;
};

// On-disk shard file (row f3; mirrors the tmp-file -> rename -> .corrupted life cycle of
// BlockManagerLocked::write_block_inner / move_block_to_corrupted, src/block/manager.rs:720-819,
// and the directory scheme data_dir/<h[0]>/<h[1]>/<hex(h)> of src/block/layout.rs:286-291):
//   <data_dir>/node<N>/<hh>/<hh>/<64 hex>.shard        64-byte header + shard bytes
// hdr_check covers the first 48 bytes (every field a reader acts on), so a flipped index /
// block_len / sum kind is caught like a flipped data byte.
struct ShardFileHeader {
    char magic[4];  // "GEC1"
    uint8_t k, m, index, sum_kind;
    uint32_t block_len;
    uint32_t shard_len;
    uint8_t sum[32];
    uint32_t hdr_check;  // Adler-32 of bytes [0, 48)
    uint8_t pad[12];     // pad[0]: LRC local groups (0 = RS, so files written before it existed read as RS); pad[1]: 1 =
                         // piggybacked RS PB(k, m), 2 = Clay(k, m) (0 = neither).  Outside hdr_check, so the reader compares them with
                         // its own code and quarantines a mismatch
};
static_assert(sizeof(ShardFileHeader) == 64, "shard file header is 64 bytes");

std::string hex_of(const uint8_t *p, size_t n)
{
    static const char *d = "0123456789abcdef";
    std::string o;
    for (size_t i = 0; i < n; i++) {
        o.push_back(d[p[i] >> 4]);
        o.push_back(d[p[i] & 15]);
    }
    return o;
}

enum ReadResult { kReadOk = 0, kReadMissing = 1, kReadInvalid = 2 };

// A run of a shard's bytes for a ranged read: the whole shard (the default), one PB half -- its length comes from the
// header read with it -- or explicit bytes [off, off + len)
struct ShardSpan {
    int half = -1;
    uint32_t off = 0, len = UINT32_MAX;  // UINT32_MAX: the whole shard
    static ShardSpan of_half(int h)
    {
        ShardSpan s;
        s.half = h;
        return s;
    }
    static ShardSpan bytes(uint32_t off, uint32_t len)
    {
        ShardSpan s;
        s.off = off;
        s.len = len;
        return s;
    }
    bool whole() const { return half < 0 && len == UINT32_MAX; }
    // [off, off + n) of a shard of L bytes; false if the span does not fit in it
    bool resolve(uint32_t L, size_t &off_out, size_t &n) const
    {
        if (half >= 0) {
            off_out = (size_t)half * (L / 2);
            n = L / 2;
        } else if (len == UINT32_MAX) {
            off_out = 0;
            n = L;
        } else {
            off_out = off;
            n = len;
        }
        return (uint64_t)off_out + n <= L;
    }
};

// the header of the shard file at `path`: kReadMissing (no such file), kReadInvalid (short, or a wrong magic or header
// check) or kReadOk.  keep != NULL: on kReadOk the open file is handed over there, positioned after the header
ReadResult read_header(const std::string &path, ShardFileHeader &hd, FILE **keep = nullptr)
{
    FILE *f = path.empty() ? nullptr : fopen(path.c_str(), "rb");  // find_block (manager.rs:627-662)
    if (!f) return kReadMissing;
    const bool ok = fread(&hd, sizeof(hd), 1, f) == 1 && memcmp(hd.magic, "GEC1", 4) == 0 &&
                    hd.hdr_check == adler32_small(reinterpret_cast<const uint8_t *>(&hd), 48);
    if (ok && keep) *keep = f;
    else fclose(f);
    return ok ? kReadOk : kReadInvalid;
}

bool fsync_dir(const std::string &dir)
{
    const int dfd = ::open(dir.c_str(), O_RDONLY | O_DIRECTORY);
    if (dfd < 0) return false;
    const bool ok = ::fsync(dfd) == 0;
    ::close(dfd);
    return ok;
}

// the whole file at `path` into `out`; false if it cannot be opened
bool read_file(const std::string &path, std::string &out)
{
    FILE *f = fopen(path.c_str(), "rb");
    if (!f) return false;
    char buf[65536];
    for (size_t r; (r = fread(buf, 1, sizeof(buf), f)) > 0;) out.append(buf, r);
    fclose(f);
    return true;
}

// `path` replaced atomically by a[0, na) + b[0, nb): a temporary file, fsynced if `fsync_file`, renamed over `path`
// (manager.rs:790-795), then the directory entry fsynced if `fsync_entry` (manager.rs:797-803).  A directory that
// cannot be opened for that fsync fails the write.  The temporary file goes on failure.
bool write_file_atomic(const std::string &path, const void *a, size_t na, const void *b, size_t nb, bool fsync_file,
                       bool fsync_entry)
{
    const std::string tmp = path + ".tmp" + std::to_string((unsigned long)::getpid());
    FILE *f = fopen(tmp.c_str(), "wb");
    if (!f) return false;
    bool ok = (na == 0 || fwrite(a, na, 1, f) == 1) && (nb == 0 || fwrite(b, nb, 1, f) == 1) && fflush(f) == 0;
    if (ok && fsync_file) ok = ::fsync(fileno(f)) == 0;  // manager.rs:775-777
    ok = (fclose(f) == 0) && ok;
    if (ok) ok = ::rename(tmp.c_str(), path.c_str()) == 0;
    if (ok && fsync_entry) ok = fsync_dir(std::filesystem::path(path).parent_path().string());
    if (!ok) ::remove(tmp.c_str());
    return ok;
}

// a code shards are stored under: RS(k, m), LRC(k, l, m - l), PB(k, m) or Clay(k, m)
struct CodeDesc {
    int k = 0, m = 0, l = 0;  // l: LRC local groups, 0 = RS
    bool pb = false;          // piggybacked RS PB(k, m): shard_len = ceil(block_len / k) rounded up to 128
    bool clay = false;        // Clay(k, m): shard_len = ceil(block_len / k) rounded up to `quantum` = 16 * alpha
    uint32_t quantum = 1;
    bool operator==(const CodeDesc &o) const { return k == o.k && m == o.m && l == o.l && pb == o.pb && clay == o.clay; }
    uint8_t kind_byte() const { return clay ? 2 : (pb ? 1 : 0); }  // header pad[1]
    bool named_by(const ShardFileHeader &hd) const { return hd.k == k && hd.m == m && hd.pad[0] == l && hd.pad[1] == kind_byte(); }
};

// A node's files for one hash (file store): <hash>.shard, written by this manager or an earlier one; <hash>.legacy,
// a shard of a previous code moved aside so that a configured-code shard can take the .shard name; <hash> (no
// extension), a whole-block replica of a replicated layout (Garage's own file: plain bytes, no header).
struct Node {
    std::mutex mu;  // stands in for the 256 hash-sharded mutexes (manager.rs:114,679-689)
    bool up = true;
    bool fsync_data = false;  // data_fsync (util/config.rs), manager.rs:775-789
    std::string dir;          // empty: in-memory store
    std::vector<CodeDesc> codes;  // [0] the configured code, then garage_bm_config.previous_codes (file store only)
    bool replicas = false;        // legacy_replicas > 0: whole-block replica files are read, listed and converted
    // the store has a layout file (DESIGN.md section 5.2): a node may hold two indices of a block, the newest version's
    // in .shard and an older version's in .legacy, and readers of a given index pick the file by its header
    std::atomic<bool> by_index{false};
    // in-memory mode: immutable shards behind shared pointers, so the node lock only covers the map operation -- the
    // 100 KB copies happen outside it (the reference shards its lock 256 ways per node, manager.rs:114,679-689; with
    // one lock per node and the copies inside it, 128 clients serialised on 14 mutexes at ~12 GiB/s)
    using ShardPtr = std::shared_ptr<const StoredShard>;
    std::unordered_map<Hash, ShardPtr, HashHasher> shards;
    std::unordered_map<Hash, ShardPtr, HashHasher> corrupted;  // the ".corrupted" quarantine
    // repair by segment (DESIGN.md section 5.15): the hashes whose quarantined copy here was quarantined because its
    // adler8 tag failed -- not named stale by the content-hash hunt or deep scrub, not a bad header.  A stale copy
    // passes its own tags, so only this verdict lets resync keep a copy's good segments.  Memory only: a restart
    // forgets it and resync rebuilds the whole shard.  Any write, erase or other quarantine of the hash clears it.
    std::unordered_set<Hash, HashHasher> tag_failed;
    // block_local_resync_queue (resync.rs:90, put_to_resync_at :241-256): one entry per hash with the time it falls
    // due (ms on the manager's clock), iterated in (due, hash) order
    std::unordered_map<Hash, int64_t, HashHasher> resync_due;
    std::set<std::pair<int64_t, Hash>> resync_queue;
    // the hash queued at `when`, or at its current due time if that is earlier
    void schedule(const Hash &h, int64_t when)
    {
        auto it = resync_due.find(h);
        if (it != resync_due.end()) {
            if (it->second <= when) return;
            resync_queue.erase({it->second, h});
            it->second = when;
        } else {
            resync_due.emplace(h, when);
        }
        resync_queue.emplace(when, h);
    }
    // resync.errors (resync.rs:605-655 ErrorCounter), plus the status of the last failure
    struct ResyncError {
        uint64_t errors = 0;
        uint64_t last_try = 0;  // ms on the manager's clock
        int32_t status = 0;
        // RESYNC_RETRY_DELAY << min(errors - 1, RESYNC_RETRY_DELAY_MAX_BACKOFF_POWER): 1 minute up to 64 minutes
        uint64_t delay_ms() const { return 60000ull << std::min<uint64_t>(errors - 1, 6); }
        uint64_t next_try() const { return last_try + delay_ms(); }
    };
    std::unordered_map<Hash, ResyncError, HashHasher> resync_errors;
    // <dir>/resync holds the queue and the error table once a scheduled step or a retry-now ran on this node (or the
    // file was there at start); resync_file_mu orders its writes
    bool resync_persist = false;
    std::mutex resync_file_mu;
    std::mutex resync_step_mu;  // one garage_bm_resync_step of this node at a time
    std::string resync_path() const { return dir + "/resync"; }
    // the file's text: format version, the queue in (due, hash) order, the error table in hash order, an Adler-32 of all
    // of that.  mu held.
    std::string resync_image() const
    {
        std::string s = "garage-bm-resync 1\n";
        for (const auto &q : resync_queue) s += "queue " + std::to_string(q.first) + " " + hex_of(q.second.data(), 32) + "\n";
        std::vector<std::pair<Hash, ResyncError>> errs(resync_errors.begin(), resync_errors.end());
        std::sort(errs.begin(), errs.end(), [](const auto &a, const auto &b) { return a.first < b.first; });
        for (const auto &e : errs)
            s += "error " + hex_of(e.first.data(), 32) + " " + std::to_string(e.second.errors) + " " +
                 std::to_string(e.second.last_try) + " " + std::to_string(e.second.status) + "\n";
        s += "check " + std::to_string(adler32_small(reinterpret_cast<const uint8_t *>(s.data()), s.size())) + "\n";
        return s;
    }
    // the queue and error table of <dir>/resync merged in (mu held): true if the file was there and read.  A file that
    // fails its check or format is ignored; garage_bm_repair_enqueue_missing finds the missing shards again.
    bool load_resync()
    {
        std::string s;
        if (dir.empty() || !read_file(resync_path(), s)) return false;
        const size_t c = s.rfind("check ");
        if (c == std::string::npos || (c > 0 && s[c - 1] != '\n')) return false;
        if (std::to_string(adler32_small(reinterpret_cast<const uint8_t *>(s.data()), c)) + "\n" != s.substr(c + 6)) return false;
        std::vector<std::string> tok;
        for (size_t i = 0; i < c;) {
            while (i < c && isspace((unsigned char)s[i])) i++;
            const size_t j = i;
            while (i < c && !isspace((unsigned char)s[i])) i++;
            if (i > j) tok.push_back(s.substr(j, i - j));
        }
        auto num = [](const std::string &t, long long lo, long long &out) {
            char *e = nullptr;
            errno = 0;
            out = strtoll(t.c_str(), &e, 10);
            return !errno && !*e && !t.empty() && out >= lo;
        };
        auto unum = [](const std::string &t, unsigned long long &out) {
            char *e = nullptr;
            errno = 0;
            out = strtoull(t.c_str(), &e, 10);
            return !errno && !*e && !t.empty() && t[0] != '-';
        };
        size_t t = 0;
        if (tok.size() < 2 || tok[t++] != "garage-bm-resync" || tok[t++] != "1") return false;
        std::vector<std::pair<int64_t, Hash>> q;
        std::vector<std::pair<Hash, ResyncError>> errs;
        while (t < tok.size()) {
            Hash h;
            long long a = 0, st = 0;
            unsigned long long b = 0;
            if (tok[t] == "queue" && t + 3 <= tok.size() && num(tok[t + 1], LLONG_MIN, a) && tok[t + 2].size() == 64 &&
                hex_to(tok[t + 2], 32, h.data())) {
                q.emplace_back(a, h);
                t += 3;
            } else if (tok[t] == "error" && t + 5 <= tok.size() && tok[t + 1].size() == 64 && hex_to(tok[t + 1], 32, h.data()) &&
                       num(tok[t + 2], 1, a) && unum(tok[t + 3], b) && num(tok[t + 4], INT32_MIN, st) && st <= INT32_MAX) {
                ResyncError e;
                e.errors = (uint64_t)a;
                e.last_try = (uint64_t)b;
                e.status = (int32_t)st;
                errs.emplace_back(h, e);
                t += 5;
            } else {
                return false;
            }
        }
        for (const auto &x : q) schedule(x.second, x.first);
        for (const auto &e : errs) resync_errors[e.first] = e.second;
        return true;
    }

    // Node is the only owner of the file scheme: the names below, the header and the placement rules of DESIGN.md
    // sections 5.1 / 5.2 / 5.7.  The files of one hash, by ShardFile:
    enum ShardFile { kShardFile = 0, kLegacyFile = 1, kReplicaFile = 2 };
    static constexpr const char *kExt[3] = {".shard", ".legacy", ""};
    // Drives (DESIGN.md section 5.7): with a drive layout the files of h live in <root>/<hh>/<hh>/ of one of `drives`,
    // the primary of h's drive partition (where every write goes) or one of its secondaries (where reads look after
    // the primary).  Drives are separate filesystems: a rename never crosses from one drive to another.  No drives:
    // every file under `dir`, as before.
    struct Drive {
        std::string path;    // as configured, relative to `dir`
        std::string root;    // dir + "/" + path, or dir for "."
        std::string marker;  // the garage-marker id recorded for it ("" = none yet)
        uint64_t capacity = 0;
        bool read_only = false;
    };
    std::vector<Drive> drives;
    std::shared_ptr<garage_drive_layout> dlayout;
    // the drives of h's partition: the primary, then the secondaries in read order
    std::vector<int> drives_of(const Hash &h) const
    {
        const int p = garage_drive_partition_of(h.data());
        uint8_t sec[GARAGE_DRIVE_MAX_DIRS];
        const int n = std::max(0, std::min(GARAGE_DRIVE_MAX_DIRS, garage_drive_layout_secondaries(dlayout.get(), p, sec, GARAGE_DRIVE_MAX_DIRS)));
        std::vector<int> r{garage_drive_layout_primary(dlayout.get(), p)};
        r.insert(r.end(), sec, sec + n);
        return r;
    }
    static std::string dir_in(const std::string &root, const Hash &h)
    {
        return root + "/" + hex_of(h.data(), 1) + "/" + hex_of(h.data() + 1, 1);
    }
    static std::string name_of(const Hash &h, const char *ext) { return hex_of(h.data(), 32) + ext; }
    // where a new file of h goes: the primary drive's directory
    std::string dir_of(const Hash &h) const { return dir_in(drives.empty() ? dir : drives[drives_of(h)[0]].root, h); }
    std::string primary_path(const Hash &h, const char *ext) const { return dir_of(h) + "/" + name_of(h, ext); }
    // the file `ext` of h: the first of the primary and the secondaries that has it, else the primary's
    std::string path_of(const Hash &h, const char *ext) const
    {
        if (drives.empty()) return primary_path(h, ext);
        for (int d : drives_of(h)) {
            const std::string p = dir_in(drives[d].root, h) + "/" + name_of(h, ext);
            if (::access(p.c_str(), F_OK) == 0) return p;
        }
        return primary_path(h, ext);
    }
    // the name `ext` of h next to the file at `path` (the same directory, so a rename to it stays on its drive)
    static std::string sibling(const std::string &path, const Hash &h, const char *ext)
    {
        return path.substr(0, path.rfind('/') + 1) + name_of(h, ext);
    }
    // the name `ext` of h removed from the primary and every secondary; true if a file was removed
    bool remove_file(const Hash &h, const char *ext)
    {
        if (drives.empty()) return ::remove(path_of(h, ext).c_str()) == 0;
        bool any = false;
        for (int d : drives_of(h)) any = ::remove((dir_in(drives[d].root, h) + "/" + name_of(h, ext)).c_str()) == 0 || any;
        return any;
    }
    // copies of the name `ext` of h other than the one at `keep`, removed: a write to the primary replaces them, as a
    // rename over the name does in one directory
    void remove_copies(const Hash &h, const char *ext, const std::string &keep)
    {
        if (drives.empty()) return;
        for (int d : drives_of(h)) {
            const std::string p = dir_in(drives[d].root, h) + "/" + name_of(h, ext);
            if (p != keep) ::remove(p.c_str());
        }
    }
    // ---- the drive layout's own files: <dir>/data_layout and a garage-marker in every drive
    uint64_t drive_gen = 0;  // bumped by every change of `drives` (a rebalance pass drops secondaries of its own layout only)
    std::string drive_layout_path() const { return dir + "/data_layout"; }
    // Garage's dir_not_empty: a garage-marker file or a hex-named subdirectory
    static bool dir_non_empty(const std::string &root)
    {
        std::error_code ec;
        if (std::filesystem::exists(root + "/garage-marker", ec)) return true;
        for (const auto &e : std::filesystem::directory_iterator(root, ec)) {
            std::error_code ec2;
            const std::string n = e.path().filename().string();
            std::vector<uint8_t> b(n.size() / 2 + 1);
            if (!n.empty() && n.size() % 2 == 0 && hex_to(n, n.size() / 2, b.data()) && e.is_directory(ec2)) return true;
        }
        return false;
    }
    // <dir>/data_layout, atomically: format version, every drive (path, capacity, read-only, marker), the layout image,
    // and an Adler-32 of all of that
    bool save_drives() const
    {
        std::string s = "garage-bm-data-layout 1\n";
        for (const Drive &d : drives) {
            s += "dir " + hex_of(reinterpret_cast<const uint8_t *>(d.path.data()), d.path.size()) + " " +
                 std::to_string(d.capacity) + " " + (d.read_only ? "1" : "0") + " " +
                 (d.marker.empty() ? std::string("-") : hex_of(reinterpret_cast<const uint8_t *>(d.marker.data()), d.marker.size())) +
                 "\n";
        }
        std::vector<uint8_t> img(garage_drive_layout_serialize(dlayout.get(), nullptr, 0));
        garage_drive_layout_serialize(dlayout.get(), img.data(), img.size());
        s += "layout " + hex_of(img.data(), img.size()) + "\n";
        s += "check " + std::to_string(adler32_small(reinterpret_cast<const uint8_t *>(s.data()), s.size())) + "\n";
        return write_file_atomic(drive_layout_path(), s.data(), s.size(), nullptr, 0, true, fsync_data);
    }
    // 1: `drives` and `dlayout` loaded from <dir>/data_layout; 0: no file; -1: a file that fails its check or format
    int load_drives()
    {
        std::string s;
        if (!read_file(drive_layout_path(), s)) return 0;
        const size_t c = s.rfind("check ");
        if (c == std::string::npos || (c > 0 && s[c - 1] != '\n')) return -1;
        if (std::to_string(adler32_small(reinterpret_cast<const uint8_t *>(s.data()), c)) + "\n" != s.substr(c + 6)) return -1;
        std::vector<std::string> tok;
        for (size_t i = 0; i < c;) {
            while (i < c && isspace((unsigned char)s[i])) i++;
            const size_t j = i;
            while (i < c && !isspace((unsigned char)s[i])) i++;
            if (i > j) tok.push_back(s.substr(j, i - j));
        }
        auto unhex = [](const std::string &h, std::string &out) {
            out.assign(h.size() / 2, '\0');
            return h.size() % 2 == 0 && hex_to(h, h.size() / 2, reinterpret_cast<uint8_t *>(&out[0]));
        };
        size_t t = 0;
        if (tok.size() < 2 || tok[t++] != "garage-bm-data-layout" || tok[t++] != "1") return -1;
        std::vector<Drive> ds;
        while (t + 5 <= tok.size() && tok[t] == "dir") {
            Drive d;
            char *e = nullptr;
            errno = 0;
            d.capacity = strtoull(tok[t + 2].c_str(), &e, 10);
            if (errno || *e || !unhex(tok[t + 1], d.path) || d.path.empty() || (tok[t + 3] != "0" && tok[t + 3] != "1")) return -1;
            d.read_only = tok[t + 3] == "1";
            if (tok[t + 4] != "-" && !unhex(tok[t + 4], d.marker)) return -1;
            d.root = root_of(d.path);
            ds.push_back(std::move(d));
            t += 5;
        }
        std::string img;
        if (t + 2 != tok.size() || tok[t] != "layout" || !unhex(tok[t + 1], img)) return -1;
        garage_drive_layout *l = nullptr;
        if (garage_drive_layout_deserialize(&l, reinterpret_cast<const uint8_t *>(img.data()), img.size()) != GARAGE_LAYOUT_OK)
            return -1;
        dlayout.reset(l, garage_drive_layout_free);
        bool ok = garage_drive_layout_n_dirs(l) == (int)ds.size();
        std::vector<uint8_t> img2(img.size());
        garage_drive_layout_serialize(l, img2.data(), img2.size());
        for (size_t i = 0; ok && i < ds.size(); i++) {  // the image's capacities are the drives'
            uint64_t cap = 0;
            memcpy(&cap, img2.data() + 5 + 8 * i, 8);
            ok = cap == (ds[i].read_only ? 0 : ds[i].capacity);
        }
        if (!ok) {
            dlayout.reset();
            return -1;
        }
        drives = std::move(ds);
        drive_gen++;
        return 1;
    }
    std::string root_of(const std::string &path) const { return path == "." ? dir : dir + "/" + path; }
    // Garage's check_markers over `ds`: a recorded marker must be in its drive's garage-marker file; a drive without one
    // records the file's, or writes a new random one.  false: a drive fails (unmounted, or another disk).
    static bool check_markers(std::vector<Drive> &ds)
    {
        for (Drive &d : ds) {
            std::string have;
            const bool found = read_file(d.root + "/garage-marker", have);
            if (!d.marker.empty()) {
                if (!found || have != d.marker) return false;
            } else if (found && !have.empty()) {
                d.marker = have;
            } else {
                std::error_code ec;
                std::filesystem::create_directories(d.root, ec);
                std::random_device rd;
                uint8_t id[16];
                for (auto &b : id) b = (uint8_t)rd();
                d.marker = hex_of(id, sizeof(id));
                if (!write_file_atomic(d.root + "/garage-marker", d.marker.data(), d.marker.size(), nullptr, 0, true, true))
                    return false;
            }
        }
        return true;
    }
    // Garage restarting with the data_dir list `cfg` (garage_bm_data_dir, checked by the caller): the layout updated
    // from the current one (initialised if there is none), markers checked, <dir>/data_layout written.  false: a marker
    // check or the write failed, and nothing changed.
    bool set_drives(const garage_bm_data_dir *cfg, int n)
    {
        std::vector<Drive> ds(n);
        std::vector<int> prev_index(n, -1);
        std::vector<uint64_t> cap(n);
        std::vector<uint8_t> non_empty(n);
        for (int i = 0; i < n; i++) {
            ds[i].path = normal_path(cfg[i].path);
            ds[i].root = root_of(ds[i].path);
            ds[i].read_only = cfg[i].read_only != 0;
            ds[i].capacity = ds[i].read_only ? 0 : cfg[i].capacity;
            cap[i] = ds[i].capacity;
            for (size_t j = 0; j < drives.size(); j++)
                if (drives[j].path == ds[i].path) {
                    prev_index[i] = (int)j;
                    ds[i].marker = drives[j].marker;
                }
            non_empty[i] = dir_non_empty(ds[i].root);
        }
        garage_drive_layout *l = nullptr;
        const int rc = dlayout ? garage_drive_layout_update(&l, dlayout.get(), prev_index.data(), n, cap.data(), non_empty.data())
                               : garage_drive_layout_init(&l, n, cap.data(), non_empty.data());
        if (rc != GARAGE_LAYOUT_OK) return false;
        std::shared_ptr<garage_drive_layout> nl(l, garage_drive_layout_free);
        if (!check_markers(ds)) return false;
        std::swap(drives, ds);
        std::swap(dlayout, nl);
        if (!save_drives()) {
            std::swap(drives, ds);
            std::swap(dlayout, nl);
            return false;
        }
        drive_gen++;
        return true;
    }
    static std::string normal_path(const char *p)
    {
        std::string s = std::filesystem::path(p).lexically_normal().string();
        while (s.size() > 1 && s.back() == '/') s.pop_back();
        return s;
    }
    // the hashes with a file on a drive that is not the primary of their partition (duplicates possible)
    void misplaced(std::vector<Hash> &out) const
    {
        for (size_t d = 0; d < drives.size(); d++) {
            std::vector<Hash> hs;
            drive_list(d, hs);
            for (const Hash &h : hs)
                if (drives_of(h)[0] != (int)d) out.push_back(h);
        }
    }
    enum MoveResult { kMoveGone = 0, kMoved, kMoveStale, kMoveQuarantined, kMoveFailed };
    // RebalanceWorker's move of file `ext` of h off drive d (not h's primary): read and checked (a shard by its header
    // and tag; a replica is moved as it is, convert_step checks its content hash), written whole to the primary, then
    // the old copy removed -- a file never changes drive by a rename.  A copy the primary already has is removed only.  A
    // shard that fails is quarantined where it is.  allow() gates the write and the removal.  *bytes: the file's size.
    MoveResult move_to_primary(const Hash &h, int d, const char *ext, const std::function<bool()> &allow, uint64_t *bytes)
    {
        const std::string from = dir_in(drives[d].root, h) + "/" + name_of(h, ext);
        std::string buf;
        if (!read_file(from, buf)) return kMoveGone;
        *bytes = buf.size();
        if (ext[0]) {
            ShardFileHeader hd;
            bool good = buf.size() >= sizeof(hd);
            if (good) memcpy(&hd, buf.data(), sizeof(hd));
            good = good && memcmp(hd.magic, "GEC1", 4) == 0 && hd.hdr_check == adler32_small(reinterpret_cast<const uint8_t *>(&hd), 48) &&
                   (uint64_t)buf.size() == sizeof(hd) + (uint64_t)hd.shard_len;
            Hash got;
            good = good && garage_ec_shard_sum_host(hd.sum_kind, reinterpret_cast<const uint8_t *>(buf.data()) + sizeof(hd),
                                                    hd.shard_len, got.data()) == GARAGE_EC_OK &&
                   memcmp(got.data(), hd.sum, 32) == 0;
            if (!good) return ::rename(from.c_str(), sibling(from, h, ".corrupted").c_str()) == 0 ? kMoveQuarantined : kMoveFailed;
        }
        const std::string to = primary_path(h, ext);
        if (::access(to.c_str(), F_OK) == 0) return allow() && ::remove(from.c_str()) == 0 ? kMoveStale : kMoveFailed;
        std::error_code ec;
        std::filesystem::create_directories(dir_of(h), ec);
        if (!allow() || !write_file_atomic(to, buf.data(), buf.size(), nullptr, 0, fsync_data, fsync_data)) return kMoveFailed;
        return allow() && ::remove(from.c_str()) == 0 ? kMoved : kMoveFailed;
    }
    // previous codes or replicas are configured (a file store changing its code)
    bool legacy_store() const { return codes.size() >= 2 || replicas; }
    // in-memory: the copy was made by the caller; the shard it replaces is returned, to be freed outside the lock
    ShardPtr store_put_ptr(const Hash &h, ShardPtr sp)
    {
        tag_failed.erase(h);
        shards[h].swap(sp);
        return sp;
    }
    ShardPtr store_find(const Hash &h) const
    {
        auto it = shards.find(h);
        return it == shards.end() ? ShardPtr() : it->second;
    }
    bool meta_valid(const ShardMeta &mt, int code = 0) const
    {
        const CodeDesc &c = codes[code];
        if (mt.index < 0 || mt.index >= c.k + c.m) return false;
        const uint64_t L = ((uint64_t)mt.block_len + (unsigned)c.k - 1) / (unsigned)c.k;
        return mt.shard_len == (L + c.quantum - 1) / c.quantum * c.quantum;
    }
    // all store_* are called with `mu` held
    // the code a shard file's header names: an index into `codes`, -1 for another code or a damaged header, -2 if the
    // file does not exist
    int file_code(const std::string &path) const
    {
        ShardFileHeader hd;
        const ReadResult r = read_header(path, hd);
        if (r == kReadMissing) return -2;
        for (size_t i = 0; r == kReadOk && i < codes.size(); i++)
            if (codes[i].named_by(hd)) return (int)i;
        return -1;
    }
    // the file holding this node's shard of `code` ("" = none).  The configured code lives in .shard; a shard of a
    // previous code in .shard (written before the code changed) or .legacy.  A file whose header names no listed code
    // is the configured code's to read, which quarantines it, as before previous codes existed.
    std::string path_for(const Hash &h, int code) const
    {
        const std::string sh = path_of(h, ".shard");
        if (codes.size() < 2) return code == 0 ? sh : std::string();
        const int c = file_code(sh);
        if (code == 0) return c >= 1 || c == -2 ? std::string() : sh;
        if (c == code) return sh;
        const std::string lg = path_of(h, ".legacy");
        const int c2 = file_code(lg);
        return c2 == code || c2 == -1 ? lg : std::string();
    }
    bool has_code(const Hash &h, int code) const { return !path_for(h, code).empty(); }
    // the shard index a configured-code file's header names: -1 for another code or a damaged header, -2 if the file
    // does not exist
    int file_index(const std::string &path) const
    {
        ShardFileHeader hd;
        const ReadResult r = read_header(path, hd);
        if (r == kReadMissing) return -2;
        return r == kReadOk && codes[0].named_by(hd) ? hd.index : -1;
    }
    // the file holding shard `index` of h ("" = none): .shard or .legacy, whichever header names that index
    std::string path_at(const Hash &h, int index) const
    {
        const std::string sh = path_of(h, ".shard"), lg = path_of(h, ".legacy");
        if (file_index(sh) == index) return sh;
        return file_index(lg) == index ? lg : std::string();
    }
    // by_index stores: h's configured-code files whose index is not `keep`, as (extension, index)
    std::vector<std::pair<const char *, int>> other_index_files(const Hash &h, int keep) const
    {
        std::vector<std::pair<const char *, int>> r;
        if (dir.empty() || !by_index) return r;
        for (const char *ext : {".shard", ".legacy"}) {
            const int i = file_index(path_of(h, ext));
            if (i >= 0 && i != keep) r.emplace_back(ext, i);
        }
        return r;
    }
    // those files removed, allow() gating each removal; the number removed
    int erase_other_indices(const Hash &h, int keep, const std::function<bool()> &allow)
    {
        int n = 0;
        for (auto &f : other_index_files(h, keep))
            if (allow() && remove_file(h, f.first)) n++;
        return n;
    }
    bool has_legacy_shard(const Hash &h) const
    {
        if (codes.size() < 2) return false;
        const int c = file_code(path_of(h, ".shard"));
        return c >= 1 || file_code(path_of(h, ".legacy")) != -2;
    }
    bool has_replica(const Hash &h) const
    {
        struct stat sb;
        return replicas && ::stat(path_of(h, "").c_str(), &sb) == 0 && S_ISREG(sb.st_mode);
    }
    // this node's legacy copies of h (a previous code's shard, the replica): removed, their number returned
    int store_erase_legacy(const Hash &h, const std::function<bool()> &allow)
    {
        int n = 0;
        if (codes.size() >= 2) {
            const std::string sh = path_of(h, ".shard"), lg = path_of(h, ".legacy");
            if (file_code(sh) >= 1 && allow() && remove_file(h, ".shard")) n++;
            if (file_code(lg) != -2 && allow() && remove_file(h, ".legacy")) n++;
        }
        if (has_replica(h) && allow() && remove_file(h, "")) n++;
        return n;
    }
    // a whole-block replica into dst (cap bytes); its length is the file size.  The caller checks the content hash.
    ReadResult replica_read_into(const Hash &h, uint8_t *dst, size_t cap, uint32_t &len) const
    {
        if (!replicas) return kReadMissing;
        FILE *f = fopen(path_of(h, "").c_str(), "rb");
        if (!f) return kReadMissing;
        struct stat sb;
        ReadResult r = kReadInvalid;
        if (fstat(fileno(f), &sb) == 0 && S_ISREG(sb.st_mode) && (uint64_t)sb.st_size <= cap && sb.st_size > 0 &&
            fread(dst, (size_t)sb.st_size, 1, f) == 1) {
            len = (uint32_t)sb.st_size;
            r = kReadOk;
        }
        fclose(f);
        return r;
    }
    // Shard mt.index of h (n bytes) stored under the configured code; the file store writes it atomically.  .shard
    // first moves to .legacy (an atomic rename, then the directory entry under data_fsync) when it holds a previous
    // code's shard (DESIGN.md section 5.1), or, in a by_index store, another index while the one written is `newest`,
    // the index the newest layout version gives this node; an older index is written to .legacy instead (section
    // 5.2).  allow() gates the move and the write, one file operation each.  false: the write did not happen.
    bool store_put(const Hash &h, const ShardMeta &mt, const uint8_t *bytes, size_t n, int newest = -1,
                   const std::function<bool()> &allow = [] { return true; })
    {
        tag_failed.erase(h);
        if (dir.empty()) {
            auto sp = std::make_shared<StoredShard>();
            static_cast<ShardMeta &>(*sp) = mt;
            sp->bytes.assign(bytes, bytes + n);
            store_put_ptr(h, std::move(sp));
            return true;
        }
        const std::string sh = path_of(h, ".shard");
        const int si = by_index ? file_index(sh) : -1;
        const bool other = si >= 0 && si != mt.index;  // .shard holds another index of h
        const bool aside = other ? mt.index == newest : codes.size() >= 2 && file_code(sh) >= 1;
        const std::string lg = sibling(sh, h, ".legacy");
        if (aside && !(allow() && ::rename(sh.c_str(), lg.c_str()) == 0 &&
                       (!fsync_data || fsync_dir(lg.substr(0, lg.rfind('/'))))))
            return false;
        if (aside) remove_copies(h, ".legacy", lg);
        if (!allow()) return false;
        std::error_code ec;
        std::filesystem::create_directories(dir_of(h), ec);
        ShardFileHeader hd;
        memset(&hd, 0, sizeof(hd));
        memcpy(hd.magic, "GEC1", 4);
        hd.k = (uint8_t)codes[0].k;
        hd.m = (uint8_t)codes[0].m;
        hd.index = (uint8_t)mt.index;
        hd.sum_kind = mt.sum_kind;
        hd.block_len = mt.block_len;
        hd.shard_len = (uint32_t)n;
        memcpy(hd.sum, mt.sum.data(), 32);
        hd.hdr_check = adler32_small(reinterpret_cast<const uint8_t *>(&hd), 48);
        hd.pad[0] = (uint8_t)codes[0].l;
        hd.pad[1] = codes[0].kind_byte();
        const char *ext = other && !aside ? ".legacy" : ".shard";
        const std::string to = primary_path(h, ext);
        if (!write_file_atomic(to, &hd, sizeof(hd), bytes, n, fsync_data, fsync_data)) return false;
        remove_copies(h, ext, to);
        return true;
    }
    // shard bytes straight into `dst` (cap bytes available), metadata into `mt`.  A span other than the whole shard
    // is one ranged read of its bytes only, into dst (which then holds the span's bytes); an empty span reads and checks
    // the header alone.  Only the node knows where a shard's bytes sit in its file.
    // index >= 0 (by_index stores): the file holding that index
    ReadResult store_read_into(const Hash &h, uint8_t *dst, size_t cap, ShardMeta &mt, ShardSpan span = {}, int code = 0,
                               int index = -1) const
    {
        if (dir.empty()) {
            auto it = code == 0 ? shards.find(h) : shards.end();
            if (it == shards.end()) return kReadMissing;
            return copy_out(*it->second, dst, cap, mt, false, span);
        }
        if (index >= 0 && by_index) return file_read_into(path_at(h, index), 0, dst, cap, mt, span);
        return file_read_into(path_for(h, code), code, dst, cap, mt, span);
    }
    // Salvage (DESIGN.md section 5.14): h's configured-code shard whole into dst, from its live file or, `quarantined`,
    // from its ".corrupted" copy (memory store: Node::corrupted).  The header is checked as on every read (file store:
    // its Adler-32 check, the code it names, its lengths); the tag is not, and nothing is moved or queued.
    ReadResult salvage_read(const Hash &h, bool quarantined, uint8_t *dst, size_t cap, ShardMeta &mt) const
    {
        if (dir.empty()) {
            const auto &map = quarantined ? corrupted : shards;
            auto it = map.find(h);
            return it == map.end() ? kReadMissing : copy_out(*it->second, dst, cap, mt);
        }
        return quarantined ? file_read_into(path_of(h, ".corrupted"), 0, dst, cap, mt) : store_read_into(h, dst, cap, mt);
    }
    // h has a quarantined copy here (".corrupted", memory store: Node::corrupted)
    bool has_quarantined(const Hash &h) const
    {
        if (dir.empty()) return corrupted.count(h) != 0;
        std::error_code ec;
        return std::filesystem::exists(path_of(h, ".corrupted"), ec);
    }
    // one shard file read as a shard of `code`
    ReadResult file_read_into(const std::string &path, int code, uint8_t *dst, size_t cap, ShardMeta &mt, ShardSpan span = {}) const
    {
        ShardFileHeader hd;
        FILE *f = nullptr;
        const ReadResult hr = read_header(path, hd, &f);
        if (hr != kReadOk) return hr;
        const CodeDesc &c = codes[code];
        ReadResult r = kReadInvalid;
        struct stat sb;
        // a header that fails any of these is a corrupt shard, never a reason to allocate or read
        // what it claims (a flipped shard_len must not become a 4 GiB resize)
        if (c.named_by(hd) && fstat(fileno(f), &sb) == 0 && (uint64_t)sb.st_size == (uint64_t)hd.shard_len + sizeof(hd)) {
            mt.index = hd.index;
            mt.block_len = hd.block_len;
            mt.shard_len = hd.shard_len;
            mt.sum_kind = hd.sum_kind;
            memcpy(mt.sum.data(), hd.sum, 32);
            size_t off = 0, n = 0;
            if (span.whole()) {
                if (meta_valid(mt, code) && mt.shard_len <= cap && (mt.shard_len == 0 || fread(dst, mt.shard_len, 1, f) == 1))
                    r = kReadOk;
            } else if ((span.half < 0 || c.pb) && meta_valid(mt, code) && span.resolve(mt.shard_len, off, n) && n <= cap &&
                       (n == 0 || ::pread(fileno(f), dst, n, (off_t)(sizeof(hd) + off)) == (ssize_t)n)) {
                r = kReadOk;
            }
        }
        fclose(f);
        return r;
    }
    ReadResult copy_out(const StoredShard &sh, uint8_t *dst, size_t cap, ShardMeta &mt, bool for_dma = false,
                        ShardSpan span = {}) const
    {
        mt = sh;
        size_t off = 0, n = 0;
        if (!meta_valid(mt) || sh.bytes.size() != mt.shard_len || !span.resolve(mt.shard_len, off, n) || n > cap ||
            (span.half >= 0 && !codes[0].pb))
            return kReadInvalid;
        if (for_dma) copy_for_dma(dst, sh.bytes.data() + off, n);
        else if (n) memcpy(dst, sh.bytes.data() + off, n);
        return kReadOk;
    }
    // the files scrub checks for h (ShardFile values): only .shard in a store without previous codes, replicas or a
    // layout file; otherwise each of .shard, .legacy and the replica that exists
    std::vector<int> scrub_files(const Hash &h) const
    {
        if (dir.empty() || !(legacy_store() || by_index)) return {kShardFile};
        std::vector<int> r;
        if (file_code(path_of(h, ".shard")) != -2) r.push_back(kShardFile);
        if (file_code(path_of(h, ".legacy")) != -2) r.push_back(kLegacyFile);
        if (has_replica(h)) r.push_back(kReplicaFile);
        return r;
    }
    // scrub's read of file (kShardFile / kLegacyFile) of h, as the code its header names.  A header naming no listed
    // code is read as the configured code (.shard) or the first previous one (.legacy), which fails it, as before
    // previous codes existed; a store with a layout file and no previous codes holds the configured code in both.
    ReadResult scrub_read_into(const Hash &h, int file, uint8_t *dst, size_t cap, ShardMeta &mt) const
    {
        if (dir.empty() || !(legacy_store() || by_index)) return store_read_into(h, dst, cap, mt);
        const std::string path = path_of(h, kExt[file]);
        return file_read_into(path, legacy_store() ? std::max(file, file_code(path)) : 0, dst, cap, mt);
    }
    // restart: the length of block h as a readable shard of any listed code on this node gives it; unless `known`
    // (another node gave it already), also an older layout version's index in .legacy, or the size of the replica (at
    // most max_len).  `tmp` holds a shard of the largest code.  false: no file gives it.
    bool block_len_of(const Hash &h, std::vector<uint8_t> &tmp, uint32_t max_len, bool known, uint32_t &len) const
    {
        ShardMeta mt;
        for (int c = 0; c < (int)codes.size(); c++)
            if (store_read_into(h, tmp.data(), tmp.size(), mt, {}, c) == kReadOk) return len = mt.block_len, true;
        if (known) return false;
        if (by_index && !legacy_store() && file_read_into(path_of(h, ".legacy"), 0, tmp.data(), tmp.size(), mt) == kReadOk)
            return len = mt.block_len, true;
        struct stat sb;
        if (has_replica(h) && ::stat(path_of(h, "").c_str(), &sb) == 0 && sb.st_size > 0 && (uint64_t)sb.st_size <= max_len)
            return len = (uint32_t)sb.st_size, true;
        return false;
    }
    bool store_get(const Hash &h, StoredShard &out) const  // a copy (scrub snapshots, inspection)
    {
        if (dir.empty()) {
            auto it = shards.find(h);
            if (it == shards.end()) return false;
            out = *it->second;
            return true;
        }
        std::error_code ec;
        const auto sz = std::filesystem::file_size(path_of(h, ".shard"), ec);
        if (ec || sz < sizeof(ShardFileHeader) || sz > (1ull << 31)) return false;
        out.bytes.resize((size_t)sz - sizeof(ShardFileHeader));
        ShardMeta mt;
        if (store_read_into(h, out.bytes.data(), out.bytes.size(), mt) != kReadOk) return false;
        static_cast<ShardMeta &>(out) = mt;
        return true;
    }
    // a configured-code shard of h is here; index >= 0: the file holding that index
    bool store_has(const Hash &h, int index = -1) const
    {
        if (dir.empty()) return shards.count(h) != 0;
        if (index >= 0) return !path_at(h, index).empty();
        if (codes.size() >= 2) return !path_for(h, 0).empty();
        std::error_code ec;
        return std::filesystem::exists(path_of(h, ".shard"), ec);
    }
    // a configured-code shard of h with this index whose header checks out is here (the stripe repair's probe, Garage's
    // NeedBlockQuery): no shard bytes are read, so a shard with bad bytes is found when it is read
    bool store_probe(const Hash &h, int index) const
    {
        if (!dir.empty()) return !path_at(h, index).empty();
        const ShardPtr sp = store_find(h);
        return sp && sp->index == index && meta_valid(*sp);
    }
    // garage_bm_block_info's look at this node's shard `index` of h (mu held, the node up): a GARAGE_BM_SHARD_* state
    // from the file header alone; nothing is quarantined or queued.  expect: the block's known length (0 = unknown).
    // Valid: the header names the configured code, this index and consistent lengths; its block length goes to
    // *block_len, and what tag_state reads goes to *tag_file (file store) or *tag_shard (memory store).
    int shard_state(const Hash &h, int index, uint32_t expect, uint32_t *block_len, std::string *tag_file,
                    ShardPtr *tag_shard) const
    {
        auto judge = [&](const ShardMeta &mt) {
            if (mt.index != index || (expect && mt.block_len != expect) || !meta_valid(mt)) return GARAGE_BM_SHARD_BAD_HEADER;
            *block_len = mt.block_len;
            return GARAGE_BM_SHARD_VALID;
        };
        if (dir.empty()) {
            const ShardPtr sp = store_find(h);
            if (!sp) return corrupted.count(h) ? GARAGE_BM_SHARD_QUARANTINED : GARAGE_BM_SHARD_ABSENT;
            if (sp->bytes.size() != sp->shard_len) return GARAGE_BM_SHARD_BAD_HEADER;
            *tag_shard = sp;
            return judge(*sp);
        }
        std::string p = by_index ? path_at(h, index) : path_for(h, 0);
        if (p.empty() && file_code(path_of(h, ".shard")) == -1) p = path_of(h, ".shard");  // a damaged or unknown header
        ShardMeta mt;
        const ReadResult r = p.empty() ? kReadMissing : file_read_into(p, 0, nullptr, 0, mt, ShardSpan::bytes(0, 0));
        if (r == kReadInvalid) return GARAGE_BM_SHARD_BAD_HEADER;
        if (r == kReadOk) {
            *tag_file = p;
            return judge(mt);
        }
        std::error_code ec;
        if (std::filesystem::exists(path_of(h, ".corrupted"), ec)) return GARAGE_BM_SHARD_QUARANTINED;
        return has_legacy_shard(h) || has_replica(h) ? GARAGE_BM_SHARD_PREVIOUS : GARAGE_BM_SHARD_ABSENT;
    }
    // The tag check of a shard shard_state found valid, without the node lock: the whole file (or the immutable
    // in-memory shard) read into `buf` (room for a shard) and its tag computed.  A file replaced meanwhile is judged as
    // it is read then.
    int tag_state(int index, uint32_t expect, const std::string &file, const ShardPtr &sp, std::vector<uint8_t> &buf) const
    {
        ShardMeta mt;
        const uint8_t *bytes = nullptr;
        if (sp) {
            mt = *sp;
            bytes = sp->bytes.data();
        } else {
            const ReadResult r = file_read_into(file, 0, buf.data(), buf.size(), mt);
            if (r == kReadMissing) return GARAGE_BM_SHARD_ABSENT;
            if (r == kReadInvalid || mt.index != index || (expect && mt.block_len != expect)) return GARAGE_BM_SHARD_BAD_HEADER;
            bytes = buf.data();
        }
        Hash got;
        if (garage_ec_shard_sum_host(mt.sum_kind, bytes, mt.shard_len, got.data()) != GARAGE_EC_OK || got != mt.sum)
            return GARAGE_BM_SHARD_BAD_TAG;
        return GARAGE_BM_SHARD_VALID;
    }
    bool store_erase(const Hash &h)
    {
        tag_failed.erase(h);
        if (dir.empty()) return shards.erase(h) != 0;
        return remove_file(h, ".shard");
    }
    // move_block_to_corrupted (manager.rs:807-819): file >= 0 that ShardFile of h; code -1 the replica; index >= 0
    // (by_index stores) the file holding that index; otherwise the file holding the shard of `code`.  tag: the shard
    // is quarantined because its adler8 tag failed (Node::tag_failed)
    void store_quarantine(const Hash &h, int code = 0, int index = -1, int file = -1, bool tag = false)
    {
        if (tag) tag_failed.insert(h);
        else tag_failed.erase(h);
        if (dir.empty()) {
            auto it = shards.find(h);
            if (it != shards.end()) {
                corrupted[h] = std::move(it->second);
                shards.erase(it);
            }
            return;
        }
        std::string p;
        if (file >= 0 || code < 0) p = path_of(h, kExt[file >= 0 ? file : kReplicaFile]);
        else if (index >= 0 && by_index) p = path_at(h, index);
        if (p.empty()) p = codes.size() < 2 ? path_of(h, ".shard") : path_for(h, code);
        if (!p.empty()) ::rename(p.c_str(), sibling(p, h, ".corrupted").c_str());
    }
    // fault injection (garage_bm_corrupt_shard*): what = 0 flips a bit of the shard's bytes at byte_off, 1 rewrites the
    // stored block_len (+1), 2 rewrites the stored index (+1 mod k+m); the stored tag / header check are left alone in
    // every case -- that is the corruption.
    int store_corrupt(const Hash &h, size_t byte_off, int what)
    {
        if (dir.empty()) {
            auto it = shards.find(h);
            if (it == shards.end()) return GARAGE_BM_E_MISSING_BLOCK;
            auto mod = std::make_shared<StoredShard>(*it->second);  // stored shards are immutable: replace by a damaged copy
            if (what == 0) {
                if (mod->bytes.empty()) return GARAGE_BM_E_MISSING_BLOCK;
                mod->bytes[byte_off % mod->bytes.size()] ^= 0x01;
            } else if (what == 1) {
                mod->block_len += 1;
            } else {
                mod->index = (mod->index + 1) % (codes[0].k + codes[0].m);
            }
            it->second = std::move(mod);
            return GARAGE_BM_OK;
        }
        FILE *f = fopen(path_of(h, ".shard").c_str(), "r+b");
        if (!f) return GARAGE_BM_E_MISSING_BLOCK;
        ShardFileHeader hd;
        int rc = GARAGE_BM_E_MISSING_BLOCK;
        if (fread(&hd, sizeof(hd), 1, f) == 1) {
            long off = -1;
            uint8_t b = 0;
            if (what == 0 && hd.shard_len) off = (long)sizeof(hd) + (long)(byte_off % hd.shard_len);
            else if (what == 1) off = offsetof(ShardFileHeader, block_len);
            else if (what == 2) off = offsetof(ShardFileHeader, index);
            if (off >= 0 && fseek(f, off, SEEK_SET) == 0 && fread(&b, 1, 1, f) == 1) {
                b = what == 0 ? (uint8_t)(b ^ 1) : (uint8_t)(b + 1);
                if (fseek(f, off, SEEK_SET) == 0 && fwrite(&b, 1, 1, f) == 1) rc = GARAGE_BM_OK;
            }
        }
        fclose(f);
        return rc;
    }
    // BlockStoreIterator (repair.rs:634-764): every hash this node holds a file of that it reads -- .shard, and with
    // previous codes or a layout file .legacy, with replicas configured the replica
    void store_list(std::vector<Hash> &out) const
    {
        if (dir.empty()) {
            for (auto &kv : shards) out.push_back(kv.first);
            return;
        }
        if (!drives.empty()) {
            for (size_t d = 0; d < drives.size(); d++) drive_list(d, out);
            std::sort(out.begin(), out.end());
            out.erase(std::unique(out.begin(), out.end()), out.end());
            return;
        }
        std::error_code ec;
        for (auto it = std::filesystem::recursive_directory_iterator(dir, ec);
             !ec && it != std::filesystem::recursive_directory_iterator(); it.increment(ec)) {
            Hash h;
            if (listed_name(*it, h)) out.push_back(h);
        }
    }
    // a file store_list lists: .shard, with previous codes or a layout file .legacy, with replicas configured the replica;
    // its hash into h
    bool listed_name(const std::filesystem::directory_entry &e, Hash &h) const
    {
        std::error_code ec;
        const std::string name = e.path().filename().string();
        const bool listed = (name.size() == 64 + 6 && name.compare(64, 6, ".shard") == 0) ||
                            ((codes.size() >= 2 || by_index) && name.size() == 64 + 7 && name.compare(64, 7, ".legacy") == 0) ||
                            (replicas && name.size() == 64 && e.is_regular_file(ec));
        return listed && hex_to(name, 32, h.data());
    }
    static bool hex_to(const std::string &s, size_t n, uint8_t *out)
    {
        auto v = [&](char c) { return c >= '0' && c <= '9' ? c - '0' : (c >= 'a' && c <= 'f' ? c - 'a' + 10 : -1); };
        if (s.size() < 2 * n) return false;
        for (size_t i = 0; i < n; i++) {
            const int hi = v(s[2 * i]), lo = v(s[2 * i + 1]);
            if (hi < 0 || lo < 0) return false;
            out[i] = (uint8_t)((hi << 4) | lo);
        }
        return true;
    }
    // the hashes with a listed file in drive d's <hh>/<hh>/ tree (duplicates possible)
    void drive_list(size_t d, std::vector<Hash> &out) const
    {
        namespace fs = std::filesystem;
        auto hex_dir = [](const fs::directory_entry &e) {
            std::error_code ec;
            const std::string n = e.path().filename().string();
            uint8_t b;
            return n.size() == 2 && hex_to(n, 1, &b) && e.is_directory(ec);
        };
        std::error_code ec;
        for (const auto &a : fs::directory_iterator(drives[d].root, ec)) {
            if (!hex_dir(a)) continue;
            std::error_code ec2;
            for (const auto &b : fs::directory_iterator(a.path(), ec2)) {
                if (!hex_dir(b)) continue;
                std::error_code ec3;
                for (const auto &f : fs::directory_iterator(b.path(), ec3)) {
                    Hash h;
                    if (listed_name(f, h)) out.push_back(h);
                }
            }
        }
    }
};

// ---------------------------------------------------------------- counting semaphore (bytes)
// mirrors buffer_kb_semaphore (manager.rs:156, 380-385)
class ByteSemaphore {
public:
    explicit ByteSemaphore(uint64_t cap) : cap_(cap), avail_(cap) {}
    void acquire(uint64_t n)
    {
        if (n > cap_) n = cap_;
        std::unique_lock<std::mutex> lk(mu_);
        cv_.wait(lk, [&] { return avail_ >= n; });
        avail_ -= n;
    }
    void release(uint64_t n)
    {
        if (n > cap_) n = cap_;
        {
            std::lock_guard<std::mutex> lk(mu_);
            avail_ += n;
        }
        cv_.notify_all();
    }

private:
    uint64_t cap_, avail_;
    std::mutex mu_;
    std::condition_variable cv_;
};
struct ByteLease {  // RAII: the bytes go back to the semaphore on every path
    ByteSemaphore &sem;
    const uint64_t n;
    ByteLease(ByteSemaphore &s, uint64_t bytes) : sem(s), n(bytes) { sem.acquire(n); }
    ~ByteLease() { sem.release(n); }
    ByteLease(const ByteLease &) = delete;
    ByteLease &operator=(const ByteLease &) = delete;
};

// ---------------------------------------------------------------- generic batcher (row f1)
template <class Item>
class Batcher {
public:
    using Run = std::function<void(int /*worker*/, std::vector<Item *> &)>;
    // `workers` dispatcher threads pull batches from one queue: while one batch is on the GPU the
    // next one is being collected (each worker owns a garage_ec context and buffers)
    Batcher(size_t max_items, unsigned linger_us, int workers, Run run, std::function<void()> on_thread_start)
        : max_(std::max<size_t>(1, max_items)), linger_(linger_us), run_(std::move(run))
    {
        for (int w = 0; w < std::max(1, workers); w++)
            th_.emplace_back([this, w, on_thread_start] {
                if (on_thread_start) on_thread_start();
                loop(w);
            });
    }
    ~Batcher()
    {
        {
            std::lock_guard<std::mutex> lk(mu_);
            stop_ = true;
        }
        cv_.notify_all();
        for (auto &t : th_) t.join();
    }
    // blocks the calling thread until its item has been processed in some batch
    int submit(Item &it)
    {
        std::future<int> f = it.done.get_future();
        {
            std::lock_guard<std::mutex> lk(mu_);
            q_.push_back(&it);
        }
        cv_.notify_all();
        return f.get();
    }
    // several items at once (one caller's whole batch): blocks until all are processed, their results in `rc`
    void submit_all(const std::vector<Item *> &items, std::vector<int> &rc)
    {
        std::vector<std::future<int>> fs;
        for (Item *it : items) fs.push_back(it->done.get_future());
        {
            std::lock_guard<std::mutex> lk(mu_);
            q_.insert(q_.end(), items.begin(), items.end());
        }
        cv_.notify_all();
        rc.resize(items.size());
        for (size_t i = 0; i < fs.size(); i++) rc[i] = fs[i].get();
    }
    uint64_t batches() const { return batches_.load(); }
    uint64_t items() const { return items_.load(); }

private:
    void loop(int w)
    {
        std::vector<Item *> batch;
        for (;;) {
            batch.clear();
            {
                std::unique_lock<std::mutex> lk(mu_);
                cv_.wait(lk, [&] { return stop_ || !q_.empty(); });
                if (stop_ && q_.empty()) return;
                // linger: give concurrent callers a moment to join the batch
                const auto deadline = Clock::now() + std::chrono::microseconds(linger_);
                while (q_.size() < max_ && !stop_) {
                    if (cv_.wait_until(lk, deadline) == std::cv_status::timeout) break;
                }
                while (!q_.empty() && batch.size() < max_) {
                    batch.push_back(q_.front());
                    q_.pop_front();
                }
            }
            if (batch.empty()) continue;  // another worker took them
            batches_++;
            items_ += batch.size();
            // nothing may escape a dispatcher thread: an exception (bad_alloc in a staging vector)
            // fails the items of this batch instead of terminating the process
            try {
                run_(w, batch);  // sets every item's promise
            } catch (...) {
                for (Item *it : batch)
                    if (!it->fulfilled) {
                        it->fulfilled = true;
                        it->done.set_value(GARAGE_EC_E_NOMEM);
                    }
            }
        }
    }
    const size_t max_;
    const unsigned linger_;
    Run run_;
    std::mutex mu_;
    std::condition_variable cv_;
    std::deque<Item *> q_;
    bool stop_ = false;
    std::atomic<uint64_t> batches_{0}, items_{0};
    std::vector<std::thread> th_;
};

// pool of pinned slots: the calling thread fills its slot (in parallel with every other caller)
// so the dispatcher's DMA runs at PCIe speed from pinned, NUMA-local memory -- in Garage proper
// the body copy of BytesBuf::take_exact (src/net/bytes_buf.rs:66-117) would land here directly
class SlotPool {
public:
    bool init(garage_ec_ctx *ctx, size_t slots, size_t slot_bytes)
    {
        ctx_ = ctx;
        slot_bytes_ = (slot_bytes + 4095) / 4096 * 4096;
        if (garage_ec_host_alloc(ctx, &base_, slots * slot_bytes_) != GARAGE_EC_OK) return false;
        for (size_t i = 0; i < slots; i++) free_.push_back(static_cast<uint8_t *>(base_) + i * slot_bytes_);
        return true;
    }
    uint8_t *acquire()
    {
        std::unique_lock<std::mutex> lk(mu_);
        cv_.wait(lk, [&] { return !free_.empty(); });
        uint8_t *p = free_.back();
        free_.pop_back();
        return p;
    }
    void release(uint8_t *p)
    {
        {
            std::lock_guard<std::mutex> lk(mu_);
            free_.push_back(p);
        }
        cv_.notify_all();  // a waiter for n slots must not swallow the wake-up a waiter for one needs
    }
    // n slots taken together: a caller never holds some while it waits for the rest (n <= the pool's size)
    std::vector<uint8_t *> acquire_n(size_t n)
    {
        std::unique_lock<std::mutex> lk(mu_);
        cv_.wait(lk, [&] { return free_.size() >= n; });
        std::vector<uint8_t *> r(free_.end() - (std::ptrdiff_t)n, free_.end());
        free_.resize(free_.size() - n);
        return r;
    }
    void release_n(const std::vector<uint8_t *> &ps)
    {
        {
            std::lock_guard<std::mutex> lk(mu_);
            free_.insert(free_.end(), ps.begin(), ps.end());
        }
        cv_.notify_all();
    }
    size_t slot_bytes() const { return slot_bytes_; }
    void destroy()
    {
        if (base_) garage_ec_host_free(ctx_, base_);
        base_ = nullptr;
    }

private:
    garage_ec_ctx *ctx_ = nullptr;
    void *base_ = nullptr;
    size_t slot_bytes_ = 0;
    std::mutex mu_;
    std::condition_variable cv_;
    std::vector<uint8_t *> free_;
};
struct SlotLease {  // RAII: a slot goes back to its pool on every path
    SlotPool &pool;
    uint8_t *p;
    explicit SlotLease(SlotPool &pl) : pool(pl), p(pl.acquire()) {}
    ~SlotLease() { pool.release(p); }
    SlotLease(const SlotLease &) = delete;
    SlotLease &operator=(const SlotLease &) = delete;
};

// pinned output buffer of one encode batch (parity rows + shard tags).  The callers of the batch
// store their shards straight out of it; the dispatcher reuses it only when they are all done.
struct EncBatchBuf {
    garage_ec_ctx *ctx = nullptr;
    void *p = nullptr;
    size_t cap = 0;
    std::mutex mu;
    std::condition_variable cv;
    int pending = 0;
    uint8_t *get(size_t n)
    {
        if (n > cap) {
            if (p) garage_ec_host_free(ctx, p);
            p = nullptr;
            cap = 0;
            const size_t want = std::max(n, (size_t)1 << 20);
            if (garage_ec_host_alloc(ctx, &p, want) != GARAGE_EC_OK) return nullptr;
            cap = want;
        }
        return static_cast<uint8_t *>(p);
    }
    void wait_idle()
    {
        std::unique_lock<std::mutex> lk(mu);
        cv.wait(lk, [&] { return pending == 0; });
    }
    void set_pending(int n)
    {
        std::lock_guard<std::mutex> lk(mu);
        pending = n;
    }
    void done_one()
    {
        bool zero;
        {
            std::lock_guard<std::mutex> lk(mu);
            zero = --pending == 0;
        }
        if (zero) cv.notify_all();
    }
    void release()
    {
        if (p) garage_ec_host_free(ctx, p);
        p = nullptr;
        cap = 0;
    }
};

struct EncodeItem {
    const uint8_t *data = nullptr;  // the block (pinned slot, or the caller's buffer for oversize blocks)
    uint32_t len = 0;
    // filled by the dispatcher: parity row i at parity + i * pstride, tags of the k+m shards
    const uint8_t *parity = nullptr;
    size_t pstride = 0;
    const uint8_t *sums = nullptr;
    EncBatchBuf *buf = nullptr;  // to be released (done_one) once the shards are stored
    // a sealed PUT (rpc_put_block_sealed): the block is sealed under `key` (NULL: stored as plaintext) and `nonce`; the
    // dispatcher fills `shards` (all k+m, `pstride` apart, kept alive by `sealed_out`) and the content address `hash`
    bool sealed = false;
    const uint8_t *key = nullptr;
    uint8_t nonce[8] = {0};
    uint8_t crc_kind = GARAGE_EC_CRC_NONE;  // the S3 checksum of the plaintext to compute (DESIGN.md 2.9); out: crc
    uint32_t crc = 0;
    std::shared_ptr<std::vector<uint8_t>> sealed_out;
    const uint8_t *shards = nullptr;
    Hash hash{};
    bool fulfilled = false;
    std::promise<int> done;
};

// A copy with re-encryption (rpc_put_block_resealed): the destination's pieces over the gathered source stripes.  The
// dispatcher fills the outputs; `out` keeps the batch's destination shards and tags alive.
struct ResealJob {
    std::vector<uint8_t *> stripes;  // one per distinct source: k+m shards, slot_stride apart (ciphertext)
    std::vector<uint8_t> present;    // k+m per source
    std::vector<uint32_t> src_len;
    std::vector<Hash> src_hash;
    std::vector<garage_ec_piece> pieces;  // src: an index into `stripes`
    const uint8_t *src_key = nullptr;     // NULL: the sources are plaintext
    const uint8_t *dst_key = nullptr;
    uint8_t nonce[8] = {0};
    uint8_t crc_kind = GARAGE_EC_CRC_NONE;  // the S3 checksum of the destination's plaintext; out: crc
    uint32_t crc = 0;
    std::vector<uint8_t> src_bad;       // out, per source
    std::vector<int32_t> src_status;    // out, per source
    std::shared_ptr<std::vector<uint8_t>> out;
    const uint8_t *shards = nullptr, *sums = nullptr;  // out: k+m shards slot_stride apart, their tags
    Hash hash{};
    uint32_t stored_len = 0;
};

struct ReconItem {
    // what the dispatcher does with the stripe, in the order a batch runs them: a ranged GET
    // (garage_ec_decode_range_stripes), an opened GET (garage_ec_open_stripes), a ranged opened GET
    // (garage_ec_open_range_stripes), a whole-shard rebuild (garage_ec_reconstruct_stripes), a copy with
    // re-encryption (garage_ec_reseal_stripes, its stripes in `reseal`)
    enum Kind { kRange, kOpen, kOpenRange, kRebuild, kReseal };
    static constexpr int kKinds = kReseal + 1;
    Kind kind = kRebuild;
    uint8_t *stripe = nullptr;  // pinned slot: k+m shards, slot_stride apart, survivors filled in by the caller
    uint32_t block_len = 0;     // the stored length: the sealed length for the opened kinds
    uint8_t present[GARAGE_EC_MAX_K + GARAGE_EC_MAX_M] = {0};  // the ranged kinds: the plan's presence map
    uint8_t want[GARAGE_EC_MAX_K + GARAGE_EC_MAX_M] = {0};     // rebuild: the shards to rebuild
    std::atomic<uint64_t> *call_us = nullptr;  // rebuild, non-NULL: also gets the wall time of the call that rebuilt it
    uint32_t off = 0, len = 0;  // the ranged kinds: bytes [off, off + len) of the block or plaintext go to `out`
    uint8_t *out = nullptr;     // the ranged kinds and open: where the bytes go
    const uint8_t *key = nullptr;  // the opened kinds
    Hash hash{};                   // open: the content address to check
    uint32_t plain_len = 0;        // open: set by the dispatcher
    ResealJob *reseal = nullptr;   // reseal
    bool fulfilled = false;
    std::promise<int> done;
};

// pinned scratch that grows on demand (owned by one thread at a time)
struct PinnedBuf {
    garage_ec_ctx *ctx = nullptr;
    void *p = nullptr;
    size_t cap = 0;
    uint8_t *get(size_t n)
    {
        if (n > cap) {
            if (p) garage_ec_host_free(ctx, p);
            p = nullptr;
            cap = 0;
            if (garage_ec_host_alloc(ctx, &p, n) != GARAGE_EC_OK) return nullptr;
            cap = n;
        }
        return static_cast<uint8_t *>(p);
    }
    void release()
    {
        if (p) garage_ec_host_free(ctx, p);
        p = nullptr;
        cap = 0;
    }
    ~PinnedBuf() { release(); }
};

// Everything one listed device runs (DESIGN.md section 5.13): the dispatcher contexts and threads of both batchers,
// one context per code for the sweeps' own calls, and the pinned memory its callers land blocks and stripes in,
// allocated on the device's NUMA node.  A call routed to a group takes its slots from the group's pools and submits to
// its batchers only, so a batch never spans devices.
struct DeviceGroup {
    static constexpr int kWorkers = 3;  // dispatcher threads per batcher (overlap PCIe / GPU / collection)
    static constexpr int kEncBufs = 4;  // pinned output buffers per dispatcher: a batch's callers store their shards
                                        // out of one while the dispatcher fills the next ones
    int device = 0;
    int numa_node = -1;  // the GPU's node (garage_ec_numa_info), -1 = unknown
    int pool_node = -1;  // the node its pools landed on
    garage_ec_ctx *enc_ctx[kWorkers] = {nullptr};  // one context (= its own staging lanes) per worker
    garage_ec_ctx *rec_ctx[kWorkers] = {nullptr};
    std::vector<garage_ec_ctx *> code_ctx;  // per code of garage_bm::codes; the first group's are the codes' own
    SlotPool put_slots;     // one block each
    SlotPool stripe_slots;  // (k+m) x slot_stride each: degraded GETs, resync workers
    EncBatchBuf enc_out[kWorkers][kEncBufs];
    int enc_next[kWorkers] = {0};
    std::unique_ptr<Batcher<EncodeItem>> enc_batcher;
    std::unique_ptr<Batcher<ReconItem>> rec_batcher;
    PinnedBuf scrub_buf;
    std::mutex scrub_mu;
    PinnedBuf deep_buf;  // the deep scrub's batch of stripes (not stripe_slots: DESIGN.md section 5.2's pool rule)
    std::mutex deep_mu;
    PinnedBuf conv_src, conv_dst, conv_blk;  // a conversion batch: old shards / replicas in, new shards + tags out
    std::mutex rebuild_mu;                   // garage_bm::rebuild_batch: one batch of the pool at a time
    std::atomic<uint64_t> queued{0};         // calls routed here that have not returned
    std::atomic<uint64_t> batches{0}, blocks{0}, bytes{0}, routed_local{0}, routed_remote{0};
    void count(size_t n_blocks, uint64_t n_bytes)  // one GPU call of the group
    {
        batches++;
        blocks += n_blocks;
        bytes += n_bytes;
    }
    // threads and pinned memory, before the contexts they use are destroyed
    void stop()
    {
        enc_batcher.reset();
        rec_batcher.reset();
        for (auto &w : enc_out)
            for (auto &eb : w) eb.release();
        for (PinnedBuf *b : {&scrub_buf, &deep_buf, &conv_src, &conv_dst, &conv_blk}) b->release();
        put_slots.destroy();
        stripe_slots.destroy();
    }
};

// The group the calling thread's GPU work goes to: set by garage_bm::Route for the length of one call, and for good
// in a group's dispatcher threads.  Keyed by the manager, as one process may run several.
struct RouteTls {
    const void *bm = nullptr;
    DeviceGroup *g = nullptr;
};
thread_local RouteTls tl_route;

struct RcEntry {
    int64_t count = 0;
    Clock::time_point zero_since{};  // when the count last dropped to 0 (BLOCK_GC_DELAY, manager.rs:49-52)
};

// One page of a resumable sweep (the scrub iterator checkpoint, repair.rs:186-193,460-464): `hs` sorted and
// deduplicated, then cut to the hashes after *cursor (NULL: from the start), at most `max` of them (0: all).
// *finished: the page reaches the end; *cursor_out: its last hash (none: *cursor, or zeros from the start).
void sweep_page(std::vector<Hash> &hs, const Hash *cursor, size_t max, Hash *cursor_out, int *finished)
{
    std::sort(hs.begin(), hs.end());
    hs.erase(std::unique(hs.begin(), hs.end()), hs.end());
    if (cursor) hs.erase(hs.begin(), std::upper_bound(hs.begin(), hs.end(), *cursor));
    const bool done = !max || hs.size() <= max;
    if (!done) hs.resize(max);
    if (finished) *finished = done ? 1 : 0;
    if (cursor_out) {
        if (!hs.empty()) *cursor_out = hs.back();
        else if (cursor) *cursor_out = *cursor;
        else cursor_out->fill(0);
    }
}

}  // namespace

// ================================================================= the manager
struct garage_bm {
    garage_bm_config cfg{};
    int k = 0, m = 0, tot = 0;
    int sum_kind = GARAGE_EC_SUM_ADLER8;
    size_t slot_stride = 0;  // stride of the largest block's shards: geometry of every stripe slot
    // one group per listed device, in list order (DESIGN.md section 5.13)
    std::vector<std::unique_ptr<DeviceGroup>> groups;
    std::atomic<uint64_t> route_rr{0};  // round robin among equally loaded candidates

    // The routing rule: the groups whose GPU is on the calling thread's NUMA node (getcpu(2)) are the candidates, all
    // groups if none is; the candidate with the fewest calls in flight wins, ties going round robin.
    DeviceGroup &pick_group()
    {
        unsigned cpu = 0, node = 0;
        const int here = syscall(SYS_getcpu, &cpu, &node, nullptr) == 0 ? (int)node : -1;
        bool local = false;
        for (const auto &g : groups) local = local || (here >= 0 && g->numa_node == here);
        const size_t n = groups.size(), start = (size_t)(route_rr++ % n);
        DeviceGroup *best = nullptr;
        for (size_t i = 0; i < n; i++) {
            DeviceGroup &g = *groups[(start + i) % n];
            if (local && g.numa_node != here) continue;
            if (!best || g.queued.load() < best->queued.load()) best = &g;
        }
        (local ? best->routed_local : best->routed_remote)++;
        return *best;
    }
    // Every call that reaches the GPU holds one: it routes the calling thread for the length of the call, so the
    // call's slots, batches and sweep buffers all come from one group.  A call made inside another (a GET's fallback,
    // a resync of a layout sync) keeps the outer call's group.
    struct Route {
        RouteTls saved;
        bool own;
        explicit Route(garage_bm &bm) : saved(tl_route), own(tl_route.bm != &bm)
        {
            if (!own) return;
            DeviceGroup &g = bm.pick_group();
            g.queued++;
            tl_route = {&bm, &g};
        }
        ~Route()
        {
            if (!own) return;
            tl_route.g->queued--;
            tl_route = saved;
        }
        Route(const Route &) = delete;
        Route &operator=(const Route &) = delete;
    };
    // the calling thread's group: its Route's, its dispatcher's, else the first
    DeviceGroup &grp() const { return tl_route.bm == this ? *tl_route.g : *groups[0]; }
    std::vector<std::unique_ptr<Node>> nodes;
    // stands in for the block_ref / rc tables (src/model/s3/block_ref_table.rs, src/block/rc.rs):
    // which blocks exist and how long they are.  Lock order: refs_mu before any Node::mu.
    std::mutex refs_mu;
    std::unordered_map<Hash, uint32_t, HashHasher> refs;
    // block reference counts (src/block/rc.rs): only blocks that went through block_incref /
    // block_decref have an entry; a block without entry is treated as needed (rc > 0)
    std::unordered_map<Hash, RcEntry, HashHasher> rc;
    std::unique_ptr<ByteSemaphore> ram;
    std::atomic<uint64_t> deep_blocks{0}, deep_skipped{0}, deep_parity_bad{0}, deep_content_errors{0}, deep_check_us{0};
    std::atomic<bool> warmed{false};
    // metrics (src/block/metrics.rs)
    std::atomic<uint64_t> bytes_written{0}, bytes_read{0}, corruption_counter{0}, resync_counter{0},
        resync_error_counter{0}, resync_recv_counter{0}, delete_counter{0}, put_calls{0}, reconstruct_calls{0},
        scrub_checked{0}, scrub_corrupt{0}, enc_gpu_us{0}, rec_gpu_us{0}, corrupt_data_errors{0}, write_errors{0},
        resync_shards_read{0}, resync_bytes_read{0}, resync_bytes_fetched{0};
    std::atomic<uint64_t> resync_deferred{0}, resync_steps{0}, resync_retry_nows{0}, resync_failed_bytes_read{0};
    std::atomic<uint64_t> convert_blocks{0}, convert_bytes_read{0}, convert_bytes_written{0}, convert_errors{0},
        convert_call_us{0}, legacy_gets{0}, legacy_deleted{0}, range_gets{0}, range_degraded{0}, range_bytes_read{0},
        range_bytes_fetched{0};
    std::atomic<uint64_t> sealed_range_gets{0}, sealed_range_degraded{0}, sealed_range_bytes_read{0},
        sealed_range_bytes_fetched{0}, sealed_range_auth_failures{0}, sealed_range_fallbacks{0}, sealed_range_us{0},
        sealed_range_call_us{0};
    std::atomic<uint64_t> sealed_puts{0}, sealed_batches{0}, opened_gets{0}, opened_auth_failures{0}, opened_fallbacks{0},
        seal_call_us{0}, open_call_us{0};
    std::atomic<uint64_t> reseal_calls{0}, reseal_batches{0}, reseal_sources{0}, reseal_bytes_read{0},
        reseal_auth_failures{0}, reseal_fallbacks{0}, reseal_us{0}, reseal_call_us{0};
    std::atomic<uint64_t> layout_shards_copied{0}, layout_shards_rebuilt{0}, layout_bytes_read{0}, layout_bytes_written{0},
        layout_deleted{0}, layout_sync_errors{0}, layout_bytes_fetched{0};
    std::atomic<uint64_t> salvage_attempts{0}, salvage_blocks{0}, salvage_failures{0}, salvage_units_rebuilt{0},
        salvage_quarantined_segments{0}, salvage_bytes_read{0}, salvage_call_us{0};
    std::atomic<uint64_t> segrep_repairs{0}, segrep_units_rebuilt{0}, segrep_bytes_read{0}, segrep_bytes_fetched{0},
        segrep_fallbacks{0}, segrep_call_us{0};
    std::atomic<uint64_t> stripe_repairs{0}, stripe_repair_shards{0}, stripe_repair_bytes_read{0},
        stripe_repair_bytes_fetched{0}, stripe_repair_bytes_written{0}, stripe_repair_errors{0}, stripe_repair_call_us{0};
    std::atomic<uint64_t> rebalance_files_moved{0}, rebalance_bytes_moved{0}, rebalance_errors{0}, drive_marker_errors{0};
    // per node: the drive layout generation + 1 a rebalance pass started from cursor NULL under (0 = none), and
    // whether that pass has left no misplaced file behind so far
    std::mutex rebalance_mu;
    std::vector<uint64_t> rebalance_gen;
    std::vector<uint8_t> rebalance_clean;

    // Bytes a rebuild from the shards `have` hands to the GPU, which is what crosses the network in Garage: the runs
    // garage_ec_read_ranges names for a Clay stripe (1/m of each helper for a lone lost shard), else what was read
    uint64_t fetched_bytes(const uint8_t *have, const uint8_t *want, uint32_t block_len, uint64_t read_bytes) const
    {
        if (!codes[0].clay) return read_bytes;
        garage_ec_range runs[(GARAGE_EC_MAX_K + GARAGE_EC_MAX_M) * 256];
        size_t n = 0;
        if (garage_ec_read_ranges(codes[0].ctx, have, want, (uint32_t)shard_len_of(block_len), runs,
                                  sizeof(runs) / sizeof(runs[0]), &n) != GARAGE_EC_OK)
            return read_bytes;
        uint64_t b = 0;
        for (size_t i = 0; i < n; i++) b += runs[i].len;
        return b;
    }
    // codes[0]: the configured code; codes[1..]: garage_bm_config.previous_codes, one context each, on the
    // first listed device (each group has its own for its GPU calls).  Shard i of every code lives on the i-th node of
    // the block's ring row.
    struct Code : CodeDesc {
        int tot = 0;
        garage_ec_ctx *ctx = nullptr;
    };
    std::vector<Code> codes;
    int legacy_rf = 0;  // garage_bm_config.legacy_replicas
    bool has_legacy() const { return codes.size() > 1 || legacy_rf > 0; }
    std::atomic<long> convert_ops_left{-1};  // garage_bm_debug_convert_stop_after: < 0 = off
    bool convert_op_allowed()
    {
        long v = convert_ops_left.load();
        while (v >= 0) {
            if (v == 0) return false;
            if (convert_ops_left.compare_exchange_weak(v, v - 1)) return true;
        }
        return true;
    }
    std::mutex convert_mu;         // one conversion batch at a time (in its group's pinned batch buffers)
    size_t shard_len_of(uint32_t block_len, int code = 0) const
    {
        uint32_t L = 0;  // a length that does not fit in 32 bits is larger than any slot: every caller rejects it
        return garage_ec_code_shard_len(codes[code].ctx, block_len, &L) == GARAGE_EC_OK ? L : SIZE_MAX;
    }
    // the nodes holding shards 0 .. tot-1 of h under `code`
    void nodes_of(const Hash &h, int code, int *out) const
    {
        if (code == 0) return storage_nodes_of(h, out);
        for (int i = 0; i < codes[code].tot; i++) out[i] = ring_node(h, i);
    }
    // the fixed ring: shard i of h on node (h[0] mod n) + i
    int ring_node(const Hash &h, int i) const { return ((int)h[0] % (int)nodes.size() + i) % (int)nodes.size(); }

    // rpc/layout/version.rs:117-137: top 8 bits of the hash -> partition -> k+m distinct nodes, shard i on the
    // i-th of them.  Each ring is a garage_layout (row f4, include/garage_placement.h): without garage_bm_config.layout
    // version 1 is partition p -> nodes (p mod n) + i, otherwise garage_layout_compute's.  During a layout change
    // (DESIGN.md section 5.2) several versions are active, oldest first; the set is replaced as a whole and readers
    // work on a snapshot of it.
    struct Layouts {
        std::vector<std::shared_ptr<garage_layout>> v;
        std::vector<std::vector<int32_t>> zone;      // per version: the spec it was computed from
        std::vector<std::vector<uint64_t>> capacity;
        const garage_layout *newest() const { return v.empty() ? nullptr : v.back().get(); }
        std::vector<const garage_layout *> raw() const
        {
            std::vector<const garage_layout *> r;
            for (auto &l : v) r.push_back(l.get());
            return r;
        }
    };
    std::shared_ptr<const Layouts> layouts_ = std::make_shared<Layouts>();
    std::shared_ptr<const Layouts> layouts() const { return std::atomic_load(&layouts_); }
    bool multi_version() const { return layouts()->v.size() > 1; }
    std::mutex layout_mu;               // apply_layout, the sync bookkeeping below and the layout file
    bool layout_file = false;           // a file store whose layout history is in <data_dir>/layout
    std::vector<uint64_t> synced;       // per node: the newest version it has completed a sync pass of
    std::vector<uint64_t> pass_version; // per node: the newest version when its current sync pass started (0 = none)
    std::vector<uint8_t> pass_clean;    // per node: that pass has left nothing to receive so far
    void storage_nodes_of(const Hash &h, int *out) const
    {
        static_assert(sizeof(int) == sizeof(int32_t), "node ids are 32-bit");
        auto ls = layouts();
        if (ls->newest() && garage_layout_nodes_of(ls->newest(), h.data(), reinterpret_cast<int32_t *>(out)) == GARAGE_LAYOUT_OK)
            return;
        for (int i = 0; i < tot; i++) out[i] = ring_node(h, i);  // more nodes than a ring row can name: the same rule
    }
    // the index the newest version gives `node` for h, -1 if none
    int newest_index(const Hash &h, int node) const
    {
        int who[64];
        storage_nodes_of(h, who);
        for (int i = 0; i < tot; i++)
            if (who[i] == node) return i;
        return -1;
    }

    void put_to_resync(int node, const Hash &h)  // manager.rs:592-605 / resync.rs:put_to_resync: due at once
    {
        Node &nd = *nodes[node];
        std::lock_guard<std::mutex> lk(nd.mu);
        nd.schedule(h, now_ms());
    }
    // now_msec() of the scheduled queue and the error table: ms since the epoch, or garage_bm_debug_set_clock_ms's time
    std::atomic<int64_t> debug_clock_ms{0};
    int64_t now_ms() const
    {
        const int64_t t = debug_clock_ms.load();
        if (t) return t;
        return std::chrono::duration_cast<std::chrono::milliseconds>(std::chrono::system_clock::now().time_since_epoch()).count();
    }

    void shard_tag(const uint8_t *bytes, size_t n, Hash &out) const
    {
        garage_ec_shard_sum_host(sum_kind, bytes, n, out.data());
    }

    // manager.rs:517-530 write_block: false if the node is down or the store failed (ENOSPC, EACCES ...).  The node
    // places the shard (Node::store_put).  counted: a conversion's or layout sync's write, whose move of another shard
    // aside and write are each one file operation of garage_bm_debug_convert_stop_after.
    bool write_shard(int node, const Hash &h, int index, uint32_t block_len, const uint8_t *bytes, size_t n,
                     const uint8_t *sum32, bool counted = false)
    {
        ShardMeta mt;
        mt.index = index;
        mt.block_len = block_len;
        mt.shard_len = (uint32_t)n;
        mt.sum_kind = (uint8_t)sum_kind;
        memcpy(mt.sum.data(), sum32, 32);
        Node &nd = *nodes[node];
        auto allow = [&] { return !counted || convert_op_allowed(); };
        bool ok;
        if (nd.dir.empty()) {
            auto sp = std::make_shared<StoredShard>();  // the copy happens before the node lock is taken
            static_cast<ShardMeta &>(*sp) = mt;
            sp->bytes.assign(bytes, bytes + n);
            Node::ShardPtr old;
            {
                std::lock_guard<std::mutex> lk(nd.mu);
                if (!nd.up) return false;
                ok = allow();
                if (ok) old = nd.store_put_ptr(h, std::move(sp));
            }
            // `old` (a replaced shard) is freed here, outside the lock
        } else {
            const int newest = nd.by_index ? newest_index(h, node) : -1;
            std::lock_guard<std::mutex> lk(nd.mu);
            if (!nd.up) return false;
            ok = nd.store_put(h, mt, bytes, n, newest, allow);
        }
        if (ok) bytes_written += n;
        else write_errors++;
        return ok;
    }

    // code -1: the node's replica of h.  index >= 0: the file holding that index (by_index stores).  file >= 0: that
    // Node::ShardFile of h.  tag_failed: a configured-code shard whose tag failed (a repair by segment may keep its good
    // segments, DESIGN.md section 5.15)
    void quarantine(int node, const Hash &h, int code = 0, int index = -1, int file = -1, bool tag_failed = false)
    {
        corruption_counter++;
        {
            Node &nd = *nodes[node];
            std::lock_guard<std::mutex> lk(nd.mu);
            nd.store_quarantine(h, code, index, file, tag_failed);
        }
        put_to_resync(node, h);
    }

    // manager.rs:554-609 read_block + read_block_from: the verified shard bytes land in `dst`.
    // A bad header or a tag mismatch quarantines the shard and queues a resync, like the reference.
    // `for_dma`: the GPU reads `dst` next (degraded GET, resync): see copy_for_dma
    // index >= 0: the node's shard of that index (several active layout versions)
    // span other than the whole shard (a PB half, or the tag span of a ranged GET): a ranged read of its bytes into
    // dst, checked against the tag segments it covers (garage_ec_check_shard_span_host); an empty span reads and checks
    // the header alone (dst may be NULL)
    bool read_shard_into(int node, const Hash &h, uint8_t *dst, size_t cap, ShardMeta &mt, bool for_dma = false, int code = 0,
                         int index = -1, ShardSpan span = {})
    {
        Node &nd = *nodes[node];
        ReadResult r;
        const uint8_t *check = dst;
        Node::ShardPtr sp;
        if (nd.dir.empty()) {
            {
                std::lock_guard<std::mutex> lk(nd.mu);
                if (!nd.up) return false;
                sp = nd.store_find(h);
            }
            r = sp ? nd.copy_out(*sp, dst, cap, mt, for_dma, span) : kReadMissing;  // the copy happens outside the node lock
            if (sp && for_dma && span.whole()) check = sp->bytes.data();  // same bytes, and these are still in the cache
        } else {
            std::lock_guard<std::mutex> lk(nd.mu);
            if (!nd.up) return false;
            r = nd.store_read_into(h, dst, cap, mt, span, code, index);
        }
        if (r == kReadMissing) return false;
        if (r == kReadOk) {
            if (!span.whole()) {
                size_t off = 0, n = 0;
                span.resolve(mt.shard_len, off, n);
                bytes_read += n;
                if (!n || garage_ec_check_shard_span_host(mt.sum_kind, dst, mt.shard_len, (uint32_t)off, (uint32_t)n,
                                                          mt.sum.data()) == GARAGE_EC_OK)
                    return true;
            } else {
                bytes_read += mt.shard_len;
                Hash got;
                if (garage_ec_shard_sum_host(mt.sum_kind, check, mt.shard_len, got.data()) == GARAGE_EC_OK && got == mt.sum)
                    return true;
            }
        }
        quarantine(node, h, code, index, -1, r == kReadOk && code == 0);  // a tag mismatch, or a bad header
        return false;
    }

    // ---- batch runners (dispatcher threads) -------------------------------------------------
    // the largest stored block: a block_size plaintext sealed (DESIGN.md section 2.6)
    uint32_t stored_max() const
    {
        uint32_t s = 0;
        return garage_ec_sealed_len(cfg.block_size, &s) == GARAGE_EC_OK ? s : cfg.block_size;
    }
    // the plaintext length of a block sealed to S bytes (DESIGN.md section 2.6: S = 8 + P + 16 n for its n chunks of at
    // most 4096 plaintext bytes and a tag each); false for an S the framing cannot hold (garage_ec_sealed_range's rule)
    static bool plain_len_of(uint32_t S, uint32_t &P)
    {
        uint32_t so, sl, c0, nch;
        if (garage_ec_sealed_range(S, 0, 0, &so, &sl, &c0, &nch) != GARAGE_EC_OK) return false;
        constexpr uint64_t kSealedChunk = 4096 + 16;
        P = (uint32_t)(S - 8 - 16 * ((S - 8 + kSealedChunk - 1) / kSealedChunk));
        return true;
    }

    static void wipe_secret(void *p, size_t n)
    {
        volatile uint8_t *v = static_cast<volatile uint8_t *>(p);
        while (n--) *v++ = 0;
    }

    // the sealed PUTs of a batch, keyed or stored as plaintext: one garage_ec_seal_blocks_crc call, each block with
    // its own checksum kind
    void run_seal(int w, std::vector<EncodeItem *> &b, bool keyed)
    {
        const size_t n = b.size();
        uint32_t max_len = 0;
        std::vector<const uint8_t *> ptrs(n);
        std::vector<uint32_t> lens(n), crcs(n, 0);
        std::vector<uint8_t> keys(keyed ? n * 32 : 0), nonces(keyed ? n * 8 : 0), kinds(n);
        for (size_t i = 0; i < n; i++) {
            ptrs[i] = b[i]->data;
            lens[i] = b[i]->len;
            kinds[i] = b[i]->crc_kind;
            max_len = std::max(max_len, b[i]->len);
            if (keyed) {
                memcpy(keys.data() + i * 32, b[i]->key, 32);
                memcpy(nonces.data() + i * 8, b[i]->nonce, 8);
            }
        }
        uint32_t max_b = max_len;
        if (keyed) garage_ec_sealed_len(max_len, &max_b);
        const size_t stride = garage_ec_stride_for((uint32_t)shard_len_of(max_b));
        std::shared_ptr<std::vector<uint8_t>> out;
        int rc = GARAGE_EC_OK;
        try {
            out = std::make_shared<std::vector<uint8_t>>(n * tot * stride + n * 32 + n * tot * 32);
        } catch (const std::bad_alloc &) {
            rc = GARAGE_EC_E_NOMEM;
        }
        uint8_t *sh = out ? out->data() : nullptr, *hashes = sh ? sh + n * tot * stride : nullptr,
                *sums = hashes ? hashes + n * 32 : nullptr;
        const auto t0 = Clock::now();
        if (rc == GARAGE_EC_OK)
            rc = garage_ec_seal_blocks_crc(grp().enc_ctx[w], ptrs.data(), lens.data(), keyed ? keys.data() : nullptr,
                                           keyed ? nonces.data() : nullptr, sh, stride, hashes, sums, kinds.data(),
                                           crcs.data(), n);
        seal_call_us += us_since(t0);
        sealed_batches++;
        if (keyed) wipe_secret(keys.data(), keys.size());
        for (size_t i = 0; i < n; i++) {
            if (rc == GARAGE_EC_OK) {
                b[i]->sealed_out = out;
                b[i]->shards = sh + i * tot * stride;
                b[i]->pstride = stride;
                b[i]->sums = sums + i * tot * 32;
                b[i]->crc = crcs[i];
                memcpy(b[i]->hash.data(), hashes + i * 32, 32);
            }
            b[i]->fulfilled = true;
            b[i]->done.set_value(rc);
        }
    }

    void run_encode(int w, std::vector<EncodeItem *> &all)
    {
        // sealed PUTs go to their own calls, as run_reconstruct keeps ranged GETs apart
        std::vector<EncodeItem *> b, keyed, unkeyed;
        uint64_t bytes = 0;
        for (EncodeItem *it : all) {
            (it->sealed ? (it->key ? keyed : unkeyed) : b).push_back(it);
            bytes += it->len;
        }
        grp().count(all.size(), bytes);
        if (!keyed.empty()) run_seal(w, keyed, true);
        if (!unkeyed.empty()) run_seal(w, unkeyed, false);
        if (b.empty()) return;
        const size_t n = b.size();
        uint32_t max_len = 0;
        std::vector<const uint8_t *> ptrs(n);
        std::vector<uint32_t> lens(n);
        for (size_t i = 0; i < n; i++) {
            ptrs[i] = b[i]->data;
            lens[i] = b[i]->len;
            max_len = std::max(max_len, b[i]->len);
        }
        const size_t stride = garage_ec_stride_for((uint32_t)shard_len_of(max_len));
        DeviceGroup &g = grp();
        EncBatchBuf &bb = g.enc_out[w][g.enc_next[w] = (g.enc_next[w] + 1) % DeviceGroup::kEncBufs];
        bb.wait_idle();  // the callers of the batch that last used this buffer have stored their shards
        uint8_t *par = bb.get(n * m * stride + n * tot * 32);
        int rc = par ? GARAGE_EC_OK : GARAGE_EC_E_NOMEM;
        uint8_t *sums = par ? par + n * m * stride : nullptr;
        const auto t0 = Clock::now();
        if (rc == GARAGE_EC_OK)
            rc = garage_ec_encode_blocks_with_sums(g.enc_ctx[w], ptrs.data(), lens.data(), n, par, sums, stride);
        enc_gpu_us += us_since(t0);
        if (rc == GARAGE_EC_OK) bb.set_pending((int)n);
        for (size_t i = 0; i < n; i++) {
            if (rc == GARAGE_EC_OK) {
                b[i]->parity = par + i * m * stride;
                b[i]->pstride = stride;
                b[i]->sums = sums + i * tot * 32;
                b[i]->buf = &bb;
            }
            b[i]->fulfilled = true;
            b[i]->done.set_value(rc);
        }
    }

    // a dispatcher batch: one call per kind of item in it
    void run_reconstruct(int w, std::vector<ReconItem *> &all)
    {
        std::vector<ReconItem *> by_kind[ReconItem::kKinds];
        uint64_t bytes = 0;
        for (ReconItem *it : all) {
            by_kind[it->kind].push_back(it);
            if (it->reseal)
                for (uint32_t l : it->reseal->src_len) bytes += l;
            else
                bytes += it->block_len;
        }
        grp().count(all.size(), bytes);
        for (auto &b : by_kind)
            if (!b.empty()) run_kind(w, b);
    }

    // The items of one kind: one garage_ec_* call on their stripe slots.  The columns every kind passes are packed
    // here; each kind adds its own, makes its call, adds the call's time to its counter and fulfils the items with its
    // verdict: an item's result when the call's rc is one the kind lists (any other rc is every item's result).
    void run_kind(int w, std::vector<ReconItem *> &b)
    {
        const size_t n = b.size();
        std::vector<uint8_t *> stripes(n), outs(n);
        std::vector<uint8_t> present(n * tot);
        std::vector<uint32_t> blen(n), offs(n), lens(n);
        std::vector<int32_t> status(n, 0);
        for (size_t i = 0; i < n; i++) {
            stripes[i] = b[i]->stripe;
            outs[i] = b[i]->out;
            blen[i] = b[i]->block_len;
            offs[i] = b[i]->off;
            lens[i] = b[i]->len;
            memcpy(present.data() + i * tot, b[i]->present, tot);
        }
        std::vector<uint8_t> keys;  // the opened kinds: wiped right after their call
        auto pack_keys = [&] {
            keys.resize(n * 32);
            for (size_t i = 0; i < n; i++) memcpy(keys.data() + i * 32, b[i]->key, 32);
        };
        int rc = GARAGE_EC_E_INVALID;
        auto fulfil = [&](bool listed, const std::function<int(size_t)> &verdict) {
            for (size_t i = 0; i < n; i++) {
                b[i]->fulfilled = true;
                b[i]->done.set_value(listed ? verdict(i) : rc);
            }
        };
        switch (b[0]->kind) {
        case ReconItem::kReseal: {  // keyed and plaintext sources cannot share one call
            for (const bool keyed : {true, false}) {
                std::vector<ReconItem *> g;
                for (ReconItem *it : b)
                    if ((it->reseal->src_key != nullptr) == keyed) g.push_back(it);
                if (!g.empty()) run_reseal(w, g, keyed);
            }
            break;
        }
        case ReconItem::kRebuild: {
            std::vector<uint8_t> want(n * tot);
            for (size_t i = 0; i < n; i++) {
                blen[i] = (uint32_t)shard_len_of(blen[i]);  // this call takes shard lengths
                memcpy(want.data() + i * tot, b[i]->want, tot);
            }
            const auto t0 = Clock::now();
            rc = garage_ec_reconstruct_stripes(grp().rec_ctx[w], stripes.data(), present.data(), want.data(), status.data(),
                                               blen.data(), slot_stride, n);
            const uint64_t us = us_since(t0);
            rec_gpu_us += us;
            std::set<std::atomic<uint64_t> *> counters;  // each extra counter gets the call's time once
            for (ReconItem *it : b)
                if (it->call_us) counters.insert(it->call_us);
            for (auto *c : counters) *c += us;
            fulfil(rc == GARAGE_EC_OK || rc == GARAGE_EC_E_UNRECOVERABLE,
                   [&](size_t i) { return status[i] ? GARAGE_BM_E_MISSING_BLOCK : GARAGE_BM_OK; });
            break;
        }
        case ReconItem::kRange: {
            const auto t0 = Clock::now();
            rc = garage_ec_decode_range_stripes(grp().rec_ctx[w], stripes.data(), present.data(), blen.data(), offs.data(),
                                                lens.data(), slot_stride, outs.data(), status.data(), n);
            rec_gpu_us += us_since(t0);
            fulfil(rc == GARAGE_EC_OK || rc == GARAGE_EC_E_UNRECOVERABLE,
                   [&](size_t i) { return status[i] ? GARAGE_BM_E_MISSING_BLOCK : GARAGE_BM_OK; });
            break;
        }
        case ReconItem::kOpen: {
            std::vector<uint8_t> hashes(n * 32), bad(n, 0);
            std::vector<uint32_t> plen(n, 0);
            for (size_t i = 0; i < n; i++) memcpy(hashes.data() + i * 32, b[i]->hash.data(), 32);
            pack_keys();
            const auto t0 = Clock::now();
            rc = garage_ec_open_stripes(grp().rec_ctx[w], stripes.data(), present.data(), blen.data(), hashes.data(), keys.data(),
                                        outs.data(), plen.data(), bad.data(), status.data(), slot_stride, n);
            open_call_us += us_since(t0);
            wipe_secret(keys.data(), keys.size());
            for (size_t i = 0; i < n; i++) b[i]->plain_len = plen[i];
            // a block that does not hash to its address is the wrong block (a stale shard): its tags say nothing about
            // the key, so the caller hunts the shard before any verdict on authentication
            fulfil(rc == GARAGE_EC_OK || rc == GARAGE_EC_E_UNRECOVERABLE || rc == GARAGE_EC_E_AUTH, [&](size_t i) {
                return status[i] == GARAGE_EC_E_UNRECOVERABLE ? GARAGE_BM_E_MISSING_BLOCK
                       : bad[i]                             ? GARAGE_BM_E_CORRUPT_DATA
                       : status[i]                          ? status[i]
                                                            : GARAGE_BM_OK;
            });
            break;
        }
        case ReconItem::kOpenRange: {
            pack_keys();
            const auto t0 = Clock::now();
            rc = garage_ec_open_range_stripes(grp().rec_ctx[w], stripes.data(), present.data(), blen.data(), keys.data(),
                                              offs.data(), lens.data(), slot_stride, outs.data(), status.data(), n);
            sealed_range_call_us += us_since(t0);
            wipe_secret(keys.data(), keys.size());
            fulfil(rc == GARAGE_EC_OK || rc == GARAGE_EC_E_UNRECOVERABLE || rc == GARAGE_EC_E_AUTH, [&](size_t i) {
                return status[i] == GARAGE_EC_E_UNRECOVERABLE ? GARAGE_BM_E_MISSING_BLOCK : status[i] ? status[i] : GARAGE_BM_OK;
            });
            break;
        }
        }
    }

    // The reseals of a batch: their sources back to back and their pieces renumbered, one
    // garage_ec_reseal_stripes_crc call with each destination's checksum kind; its status per destination is each
    // item's result (any other rc is every item's).  The destination shards and tags stay in one buffer the items share.
    // The dispatcher's copies of the keys are wiped after the call.
    void run_reseal(int w, std::vector<ReconItem *> &g, bool keyed)
    {
        const size_t n = g.size();
        std::vector<uint8_t *> stripes;
        std::vector<uint8_t> present, shash, skeys, dkeys(n * 32), nonces(n * 8), kinds(n);
        std::vector<uint32_t> slen, start(1, 0), crcs(n, 0);
        std::vector<garage_ec_piece> pieces;
        std::vector<size_t> base(n);
        for (size_t i = 0; i < n; i++) {
            const ResealJob &J = *g[i]->reseal;
            base[i] = stripes.size();
            for (size_t j = 0; j < J.stripes.size(); j++) {
                stripes.push_back(J.stripes[j]);
                slen.push_back(J.src_len[j]);
                shash.insert(shash.end(), J.src_hash[j].begin(), J.src_hash[j].end());
                if (keyed) skeys.insert(skeys.end(), J.src_key, J.src_key + 32);
            }
            present.insert(present.end(), J.present.begin(), J.present.end());
            for (const garage_ec_piece &p : J.pieces) pieces.push_back({(uint32_t)(base[i] + p.src), p.offset, p.len});
            start.push_back((uint32_t)pieces.size());
            memcpy(dkeys.data() + i * 32, J.dst_key, 32);
            memcpy(nonces.data() + i * 8, J.nonce, 8);
            kinds[i] = J.crc_kind;
        }
        const size_t ns = stripes.size(), sh_bytes = n * tot * slot_stride;
        auto out = std::make_shared<std::vector<uint8_t>>(sh_bytes + n * tot * 32 + n * 32);
        uint8_t *dsh = out->data(), *dsums = dsh + sh_bytes, *dhash = dsums + n * tot * 32;
        std::vector<uint32_t> dlen(n, 0);
        std::vector<uint8_t> bad(ns, 0);
        std::vector<int32_t> sst(ns, 0), st(n, 0);
        const auto t0 = Clock::now();
        const int rc = garage_ec_reseal_stripes_crc(grp().rec_ctx[w], stripes.data(), present.data(), slen.data(),
                                                    shash.data(), keyed ? skeys.data() : nullptr, ns, pieces.data(),
                                                    start.data(), dkeys.data(), nonces.data(), dsh, dhash, dsums,
                                                    dlen.data(), bad.data(), sst.data(), st.data(), kinds.data(),
                                                    crcs.data(), slot_stride, n);
        reseal_call_us += us_since(t0);
        reseal_batches++;
        wipe_secret(skeys.data(), skeys.size());
        wipe_secret(dkeys.data(), dkeys.size());
        const bool listed = rc == GARAGE_EC_OK || rc == GARAGE_EC_E_UNRECOVERABLE || rc == GARAGE_EC_E_AUTH;
        for (size_t i = 0; i < n; i++) {
            ResealJob &J = *g[i]->reseal;
            const size_t nj = J.stripes.size();
            J.src_bad.assign(bad.begin() + base[i], bad.begin() + base[i] + nj);
            J.src_status.assign(sst.begin() + base[i], sst.begin() + base[i] + nj);
            if (listed && !st[i]) {
                J.out = out;
                J.shards = dsh + i * tot * slot_stride;
                J.sums = dsums + i * tot * 32;
                memcpy(J.hash.data(), dhash + i * 32, 32);
                J.stored_len = dlen[i];
                J.crc = crcs[i];
            }
            g[i]->fulfilled = true;
            g[i]->done.set_value(listed ? st[i] : rc);
        }
    }

    // The sources of every index of h's stripe of `code`, in the order to try them, and per index a cursor on the next
    // one: with several active layout versions (code 0) the sources garage_layout_read_plan lists, each read for its file
    // of that index (by_index); else the index's ring node.  Node `skip` is left out of the indices `skip_for` names
    // (NULL: of every index).
    struct ShardSources {
        int src[GARAGE_EC_MAX_K + GARAGE_EC_MAX_M][GARAGE_BM_MAX_LAYOUT_VERSIONS];
        int nsrc[GARAGE_EC_MAX_K + GARAGE_EC_MAX_M] = {0}, cur[GARAGE_EC_MAX_K + GARAGE_EC_MAX_M] = {0};
        bool by_index = false;
        bool left(int i) const { return cur[i] < nsrc[i]; }  // a source of index i is left to try
        int node(int i) const { return src[i][cur[i]]; }
        int file(int i) const { return by_index ? i : -1; }  // the index argument of read_shard_into and quarantine
        void next(int i) { cur[i]++; }
    };
    ShardSources shard_sources(const Hash &h, int code, int skip = -1, const uint8_t *skip_for = nullptr)
    {
        const int k = codes[code].k, tot = codes[code].tot;
        ShardSources s;
        auto add = [&](int i, int node) {
            if (i < tot && s.nsrc[i] < GARAGE_BM_MAX_LAYOUT_VERSIONS && !(node == skip && (!skip_for || skip_for[i])))
                s.src[i][s.nsrc[i]++] = node;
        };
        auto ls = layouts();
        if (code == 0 && ls->v.size() > 1) {
            garage_shard_source plan[(GARAGE_EC_MAX_K + GARAGE_EC_MAX_M) * GARAGE_BM_MAX_LAYOUT_VERSIONS];
            const auto act = ls->raw();
            const int np = garage_layout_read_plan(act.data(), (int)act.size(), nullptr, 0, h.data(), k, -1, nullptr, plan,
                                                   (int)(sizeof(plan) / sizeof(plan[0])));
            for (int x = 0; x < np; x++) add(plan[x].index, plan[x].node);
            s.by_index = true;
            return s;
        }
        int who[64];
        nodes_of(h, code, who);
        for (int i = 0; i < tot; i++) add(i, who[i]);
        return s;
    }

    // Read the valid shards of `h` from every up node except `skip_node` into the stripe slot
    // (shard i at slot + i*slot_stride).  GET (want_in NULL): data shards first (a complete set needs no
    // GPU), then the survivors garage_ec_read_set names for the missing data shards -- for RS the first
    // parity shards up to k; the reference likewise stops at the first good copy (manager.rs:292-334).
    // Resync (want_in = this node's shard): exactly the read set, k/l shards for an LRC local repair.
    // PB: the halves garage_ec_read_plan names (a half at slot + i*slot_stride + half*shard_len/2, one ranged read
    // each, checked against its 4 adler8 segment tags), k + |G_i| halves for one lost data shard.
    // A shard that cannot be read is taken out of the assumed-present set and the read set recomputed.
    // A shard whose header disagrees with the others on the block length, or that sits under the
    // wrong index, is treated like a corrupt one.  `all`: read every shard (corruption hunting).
    // Returns the number of shards read (*bytes_out += the bytes); *ok = the wanted shards can be rebuilt from `have`.
    // `code`: the stripe of that code (0 = the configured one; others: a previous code's shards, moved aside or not)
    // With several active layout versions (code 0) every index has the sources garage_layout_read_plan lists for it,
    // tried in its order (a source whose file is missing or bad makes way for the next one; a PB shard's halves come
    // from one source); the wanted indices of skip_node are not read.  from_out[i] = the node shard i came from.
    int gather_into(const Hash &h, int skip_node, uint8_t *slot, uint8_t *have, uint32_t &block_len, bool all = false,
                    bool for_gpu = false, const uint8_t *want_in = nullptr, bool *ok = nullptr, uint64_t *bytes_out = nullptr,
                    int code = 0, int *from_out = nullptr)
    {
        const Code &cd = codes[code];
        const int k = cd.k, tot = cd.tot;
        const bool pb = cd.pb;
        garage_ec_ctx *const ec = cd.ctx;
        // what to read of each shard: halves (bit 0 a, bit 1 b) from garage_ec_read_plan; Clay: whole shards of
        // garage_ec_read_set (each holder checks its whole shard's tag; only the garage_ec_read_ranges runs of it are
        // handed to the rebuild)
        auto plan = [&](const uint8_t *pr, const uint8_t *wn, uint8_t *rd) {
            if (!cd.clay) return garage_ec_read_plan(ec, pr, wn, rd);
            const int rc = garage_ec_read_set(ec, pr, wn, rd);
            for (int i = 0; i < tot; i++) rd[i] = rd[i] ? 3 : 0;
            return rc;
        };
        ShardSources srcs = shard_sources(h, code, skip_node, want_in);
        memset(have, 0, tot);
        uint32_t expect = 0;
        bool have_expect = false;
        {
            std::lock_guard<std::mutex> lk(refs_mu);
            auto it = refs.find(h);
            if (it != refs.end()) {
                expect = it->second;
                have_expect = true;
            }
        }
        int count = 0;
        uint64_t nbytes = 0;
        uint8_t have_h[GARAGE_EC_MAX_K + GARAGE_EC_MAX_M] = {0};  // halves held: bit 0 a, bit 1 b (3 = whole shard)
        // whole shard (half < 0) or one half of it
        auto try_shard = [&](int i, int half = -1) {
            if (!srcs.left(i) || have_h[i] == 3) return;
            const int node = srcs.node(i), fidx = srcs.file(i);
            ShardMeta mt;
            uint8_t *dst = slot + (size_t)i * slot_stride;
            bool got;
            if (half < 0) {
                got = read_shard_into(node, h, dst, slot_stride, mt, for_gpu, code, fidx);
            } else {
                const size_t hl = (have_expect ? shard_len_of(expect, code) : slot_stride) / 2;  // placement of the b-half
                got = read_shard_into(node, h, dst + (size_t)half * hl, slot_stride - (size_t)half * hl, mt, for_gpu, code,
                                      fidx, ShardSpan::of_half(half));
                if (got && !have_expect && half == 1 && mt.shard_len / 2 != hl)  // first read of the block: move it
                    memmove(dst + mt.shard_len / 2, dst + hl, mt.shard_len / 2);
            }
            if (!got) {
                if (have_h[i]) {  // the other half came from a shard that turned out bad: drop the shard
                    have_h[i] = 0;
                    have[i] = 0;
                    count--;
                }
                srcs.next(i);
                return;
            }
            if (mt.index != i || (have_expect && mt.block_len != expect)) {
                quarantine(node, h, code, fidx);  // a stale or misplaced shard with a self-consistent tag
                if (have_h[i]) count--;
                have_h[i] = 0;
                have[i] = 0;
                srcs.next(i);
                return;
            }
            if (from_out) from_out[i] = node;
            if (!have_expect) {
                expect = mt.block_len;
                have_expect = true;
            }
            nbytes += half < 0 ? mt.shard_len : mt.shard_len / 2;
            if (!have_h[i]) count++;
            have_h[i] |= half < 0 ? 3 : (uint8_t)(1 << half);
            have[i] = 1;
        };
        uint8_t want[GARAGE_EC_MAX_K + GARAGE_EC_MAX_M] = {0};
        auto attempt = [&](int i) {  // whole shard i from its sources in order, until one is good
            do try_shard(i);
            while (!have[i] && srcs.left(i));
        };
        if (all) {
            for (int i = 0; i < tot; i++) attempt(i);
        } else {
            if (want_in) {
                memcpy(want, want_in, tot);
            } else {
                for (int i = 0; i < k; i++) {
                    attempt(i);
                    for_gpu |= !have[i];  // a data shard is missing: this stripe goes through the GPU
                    want[i] = !have[i];
                }
            }
            for (;;) {
                // assume every shard with a source not yet tried is there, a wanted one excepted; fetch what the read
                // plan still lacks (RS / LRC: whole shards of the read set; PB: the planned halves)
                uint8_t guess[GARAGE_EC_MAX_K + GARAGE_EC_MAX_M], rd[GARAGE_EC_MAX_K + GARAGE_EC_MAX_M];
                for (int i = 0; i < tot; i++) guess[i] = have[i] || (!want[i] && srcs.left(i));
                if (plan(guess, want, rd) != GARAGE_EC_OK) break;
                bool fetched = false, missing = false;
                for (int i = 0; i < tot; i++) {
                    const int need = rd[i] & ~have_h[i];
                    if (!need) continue;
                    missing = true;
                    fetched = true;
                    if (!pb || (need == 3 && !have_h[i])) {
                        attempt(i);
                    } else {
                        for (int half = 0; half < 2; half++) {
                            if (!((need >> half) & 1)) continue;
                            try_shard(i, half);
                            if (!((have_h[i] >> half) & 1)) break;  // unreadable: the shard is out, re-plan
                        }
                    }
                }
                if (!missing || !fetched) break;
            }
        }
        if (ok) {
            uint8_t rd[GARAGE_EC_MAX_K + GARAGE_EC_MAX_M];
            if (all)
                for (int i = 0; i < k; i++) want[i] = !have[i];
            *ok = plan(have, want, rd) == GARAGE_EC_OK;
            for (int i = 0; i < tot && *ok; i++) *ok = (rd[i] & ~have_h[i]) == 0;  // every planned half is here
        }
        if (bytes_out) *bytes_out += nbytes;
        block_len = expect;
        return count;
    }

    int reconstruct_in_slot(uint8_t *slot, uint32_t block_len, const uint8_t *have, const uint8_t *want, int code = 0)
    {
        reconstruct_calls++;
        if (code != 0) {  // a previous code's stripe (legacy GET): one stripe, straight on that code's context
            const uint32_t L = (uint32_t)shard_len_of(block_len, code);
            int32_t st = 0;
            const auto t0 = Clock::now();
            DeviceGroup &g = grp();
            int rc = garage_ec_reconstruct_stripes(g.code_ctx[code], &slot, have, want, &st, &L, slot_stride, 1);
            rec_gpu_us += us_since(t0);
            g.count(1, block_len);
            if (rc == GARAGE_EC_OK || rc == GARAGE_EC_E_UNRECOVERABLE) rc = st ? GARAGE_BM_E_MISSING_BLOCK : GARAGE_BM_OK;
            return rc;
        }
        ReconItem it;
        it.stripe = slot;
        it.block_len = block_len;
        memcpy(it.present, have, tot);
        memcpy(it.want, want, tot);
        return grp().rec_batcher->submit(it);
    }

    void assemble(const uint8_t *slot, uint32_t block_len, uint8_t *out, int code = 0) const
    {
        const size_t L = shard_len_of(block_len, code);
        for (int j = 0; j < codes[code].k; j++) {
            const size_t off = (size_t)j * L;
            if (off >= block_len) break;
            memcpy(out + off, slot + (size_t)j * slot_stride, std::min(L, (size_t)block_len - off));
        }
    }

    bool content_ok(const Hash &h, const uint8_t *data, size_t len) const
    {
        if (!cfg.verify_content_hash) return true;
        Hash got;
        garage_ec_blake2sum(data, len, got.data());  // DataBlock::verify, src/block/block.rs:69-83
        return got == h;
    }

    int rpc_put_block(const Hash &h, const uint8_t *data, size_t len)
    {
        Route route(*this);
        if (len == 0 || len > cfg.block_size) return GARAGE_BM_E_MESSAGE;  // blocks are at most block_size (put.rs:583-617)
        // DataBlock::from_buffer (manager.rs:376): compression is 'none' in this mirror
        ByteLease permit(*ram, (uint64_t)len * tot / k);  // manager.rs:380-385, x (k+m)/k for the parity
        put_calls++;
        // land the block in pinned memory (caller's thread, so copies of concurrent PUTs overlap)
        SlotLease slot(grp().put_slots);
        copy_for_dma(slot.p, data, len);  // landing copy: the GPU reads the slot next
        EncodeItem it;
        it.data = slot.p;
        it.len = (uint32_t)len;
        int rc = grp().enc_batcher->submit(it);
        if (rc != GARAGE_EC_OK) return rc;
        struct BufRelease {
            EncBatchBuf *b;
            ~BufRelease() { b->done_one(); }
        } rel{it.buf};
        const size_t L = shard_len_of((uint32_t)len);
        std::vector<uint8_t> pad;
        auto shard_bytes = [&](int i) -> const uint8_t * {  // valid until the next call
            if (i >= k) return it.parity + (size_t)(i - k) * it.pstride;
            const size_t off = (size_t)i * L;
            const size_t have = off < len ? std::min(L, len - off) : 0;
            if (have == L) return slot.p + off;
            pad.assign(L, 0);  // zero padded tail shard (put.rs:611-615 short last block)
            if (have) memcpy(pad.data(), slot.p + off, have);
            return pad.data();
        };
        return store_block(h, (uint32_t)len, L, shard_bytes, it.sums);
    }
    // the k+m shards of a block of len stored bytes: every active layout version, the write quorum, the block's ref
    int store_block(const Hash &h, uint32_t len, size_t L, const std::function<const uint8_t *(int)> &shard_bytes,
                    const uint8_t *sums)
    {
        int who[64];
        storage_nodes_of(h, who);  // manager.rs:373
        const int quorum = garage_ec_write_quorum(k, m, GARAGE_CONSISTENT);  // k+1 capped at k+m (row f4, garage_placement.h)
        auto ls = layouts();
        if (ls->v.size() > 1) return put_many_sets(*ls, h, len, L, shard_bytes, sums, quorum);
        int stored = 0;
        for (int i = 0; i < tot; i++)  // try_write_many_sets (manager.rs:395-405): all at once
            // only a shard that is durably stored counts towards the quorum
            if (write_shard(who[i], h, i, len, shard_bytes(i), L, sums + (size_t)i * 32)) stored++;
        {
            std::lock_guard<std::mutex> lk(refs_mu);
            refs[h] = len;
        }
        return stored >= quorum ? GARAGE_BM_OK : GARAGE_BM_E_QUORUM;
    }

    // An SSE-C PUT (put.rs:441-466): the plaintext (up to block_size bytes) lands in a put slot and goes through the
    // encode batcher, whose sealed items become one garage_ec_seal_blocks call; key NULL stores it as plaintext.  The
    // nonce prefix is 8 bytes of getrandom(2) (Garage: OsRng).  The k+m shards are stored as rpc_put_block stores a
    // block of sealed_len bytes; *hash_out = the block's content address.  crc_kind (GARAGE_EC_CRC_*): *crc_out = the
    // S3 checksum of the plaintext, from the same seal call.
    int rpc_put_block_sealed(const uint8_t *key, const uint8_t *data, size_t len, uint8_t *hash_out,
                             uint8_t crc_kind = GARAGE_EC_CRC_NONE, uint32_t *crc_out = nullptr)
    {
        Route route(*this);
        if (len > cfg.block_size || (!key && len == 0)) return GARAGE_BM_E_MESSAGE;
        uint32_t blen = (uint32_t)len;
        if (key && garage_ec_sealed_len((uint32_t)len, &blen) != GARAGE_EC_OK) return GARAGE_BM_E_MESSAGE;
        ByteLease permit(*ram, (uint64_t)blen * tot / k);
        SlotLease slot(grp().put_slots);
        if (len) copy_for_dma(slot.p, data, len);
        EncodeItem it;
        it.data = slot.p;
        it.len = (uint32_t)len;
        it.sealed = true;
        it.key = key;
        it.crc_kind = crc_kind;
        for (size_t got = 0; key && got < sizeof(it.nonce);) {
            const ssize_t r = getrandom(it.nonce + got, sizeof(it.nonce) - got, 0);
            if (r < 0 && errno != EINTR) return GARAGE_BM_E_MESSAGE;
            if (r > 0) got += (size_t)r;
        }
        const int rc = grp().enc_batcher->submit(it);
        if (rc != GARAGE_EC_OK) return rc;
        sealed_puts++;
        memcpy(hash_out, it.hash.data(), 32);
        if (crc_out) *crc_out = it.crc;
        const uint8_t *sh = it.shards;
        const size_t stride = it.pstride;
        return store_block(it.hash, blen, shard_len_of(blen), [&](int i) { return sh + (size_t)i * stride; }, it.sums);
    }

    // A copy with re-encryption into an SSE-C block (handle_copy_reencrypt, copy.rs:320-349; UploadPartCopy,
    // copy.rs:506-636; DESIGN.md section 5.11).  Each distinct source is gathered once, as rpc_get_block_opened gathers,
    // into a buffer of its own (the sources count against the RAM budget); one garage_ec_reseal_stripes call of the
    // reconstruct dispatchers proves the sources and seals the destination.  A source that the configured stripe cannot
    // serve (a previous code, replicas) or that does not hash to its address is read by rpc_get_block -- the stale-shard
    // hunt quarantines the culprit -- and its stored bytes (ciphertext for keyed sources) are framed into its buffer with
    // every data shard present; the copy is retried once.  No plaintext is in host memory on any path.  The result is
    // stored as rpc_put_block stores a block of its sealed length; refcounts are not touched.  crc_kind: *crc_out = the
    // S3 checksum of the destination's plaintext, from the GPU call that sealed it (the retry's, after a fallback).
    int rpc_put_block_resealed(const garage_bm_piece *in, int n_in, const uint8_t *src_key, const uint8_t *dst_key,
                               uint8_t *hash_out, uint32_t *stored_len_out, uint8_t crc_kind = GARAGE_EC_CRC_NONE,
                               uint32_t *crc_out = nullptr)
    {
        Route route(*this);
        const auto t0 = Clock::now();
        struct AddTime {
            std::atomic<uint64_t> &c;
            Clock::time_point t;
            ~AddTime() { c += us_since(t); }
        } add_time{reseal_us, t0};
        reseal_calls++;
        uint64_t total = 0;
        ResealJob J;
        std::vector<Hash> hs;
        for (int p = 0; p < n_in; p++) {
            if (!in[p].len) return GARAGE_EC_E_INVALID;
            total += in[p].len;
            const Hash h = to_hash(in[p].hash);
            const size_t j = std::find(hs.begin(), hs.end(), h) - hs.begin();
            if (j == hs.size()) hs.push_back(h);
            J.pieces.push_back({(uint32_t)j, in[p].offset, in[p].len});
        }
        if (total > cfg.block_size) return GARAGE_EC_E_INVALID;
        const size_t ns = hs.size(), sbytes = (size_t)tot * slot_stride;
        ByteLease permit(*ram, (uint64_t)(ns + 1) * sbytes);  // the source buffers and the destination's shards
        std::vector<std::unique_ptr<uint8_t[]>> bufs(ns);
        J.stripes.resize(ns);
        J.present.assign(ns * tot, 0);
        J.src_len.assign(ns, 0);
        J.src_hash = hs;
        J.src_key = src_key;
        J.dst_key = dst_key;
        J.crc_kind = crc_kind;
        // the stored block through rpc_get_block, framed into the source's buffer with all data shards present
        auto frame = [&](size_t j) -> int {
            reseal_fallbacks++;
            std::vector<uint8_t> blk(stored_max());
            size_t blen = 0;
            const int rc = rpc_get_block(hs[j], blk.data(), blk.size(), &blen);
            if (rc != GARAGE_BM_OK) return rc;
            reseal_bytes_read += blen;
            const size_t L = shard_len_of((uint32_t)blen);
            uint8_t *slot = J.stripes[j];
            memset(&J.present[j * tot], 0, tot);
            for (int i = 0; i < k; i++) {
                J.present[j * tot + i] = 1;
                uint8_t *row = slot + (size_t)i * slot_stride;
                memset(row, 0, slot_stride);
                const size_t off = (size_t)i * L;
                if (off < blen) memcpy(row, blk.data() + off, std::min(L, blen - off));
            }
            J.src_len[j] = (uint32_t)blen;
            return GARAGE_BM_OK;
        };
        for (size_t j = 0; j < ns; j++) {
            bufs[j].reset(new (std::nothrow) uint8_t[sbytes]);
            if (!bufs[j]) return GARAGE_EC_E_NOMEM;
            J.stripes[j] = bufs[j].get();
            bool ok = false;
            uint64_t bytes = 0;
            uint32_t bl = 0;
            gather_into(hs[j], -1, J.stripes[j], &J.present[j * tot], bl, false, false, nullptr, &ok, &bytes);
            reseal_sources++;
            reseal_bytes_read += bytes;
            J.src_len[j] = bl;
            if (!ok) {
                const int rc = frame(j);
                if (rc != GARAGE_BM_OK) return rc;
            }
        }
        for (const garage_ec_piece &p : J.pieces) {  // a source the framing cannot hold fails AUTH on the GPU
            uint32_t P = J.src_len[p.src];
            if ((!src_key || plain_len_of(P, P)) && (uint64_t)p.offset + p.len > P) return GARAGE_EC_E_INVALID;
        }
        for (size_t got = 0; got < sizeof(J.nonce);) {
            const ssize_t r = getrandom(J.nonce + got, sizeof(J.nonce) - got, 0);
            if (r < 0 && errno != EINTR) return GARAGE_BM_E_MESSAGE;
            if (r > 0) got += (size_t)r;
        }
        int rc = GARAGE_BM_OK;
        for (int attempt = 0; attempt < 2; attempt++) {
            ReconItem it;
            it.kind = ReconItem::kReseal;
            it.reseal = &J;
            rc = grp().rec_batcher->submit(it);
            if (rc != GARAGE_EC_E_UNRECOVERABLE || attempt) break;
            // a source that does not hash to its address, or that its stripe cannot rebuild: once through rpc_get_block
            bool again = false;
            for (size_t j = 0; j < ns && j < J.src_bad.size(); j++)
                if (J.src_bad[j] || J.src_status[j] == GARAGE_EC_E_UNRECOVERABLE) {
                    const int r = frame(j);
                    if (r != GARAGE_BM_OK) return r;
                    again = true;
                }
            if (!again) break;
        }
        if (rc == GARAGE_EC_E_AUTH) reseal_auth_failures++;
        if (rc == GARAGE_EC_E_UNRECOVERABLE) return GARAGE_BM_E_MISSING_BLOCK;
        if (rc != GARAGE_BM_OK) return rc;
        memcpy(hash_out, J.hash.data(), 32);
        if (stored_len_out) *stored_len_out = J.stored_len;
        if (crc_out) *crc_out = J.crc;
        const uint8_t *sh = J.shards;
        const size_t stride = slot_stride;
        return store_block(J.hash, J.stored_len, shard_len_of(J.stored_len), [&](int i) { return sh + (size_t)i * stride; },
                           J.sums);
    }

    // One opened GET of the stripe in `slot` (its shards `have`, the stored length block_len) through the reconstruct
    // dispatchers
    int open_in_slot(const Hash &h, const uint8_t *key, uint8_t *slot, uint32_t block_len, const uint8_t *have, uint8_t *out,
                     size_t cap, size_t *out_len)
    {
        uint32_t plain = 0;
        if (plain_len_of(block_len, plain) && plain > cap) return GARAGE_EC_E_INVALID;
        ReconItem it;
        it.kind = ReconItem::kOpen;
        it.stripe = slot;
        it.block_len = block_len;
        memcpy(it.present, have, tot);
        it.key = key;
        it.hash = h;
        it.out = out;
        const int rc = grp().rec_batcher->submit(it);
        if (rc == GARAGE_BM_OK) {
            opened_gets++;
            *out_len = it.plain_len;
        } else if (rc == GARAGE_EC_E_AUTH) {
            opened_auth_failures++;
        }
        return rc;
    }

    // An SSE-C GET (EncryptionParams::get_block, encryption.rs:269-279): gathered like rpc_get_block, then the rebuild,
    // the content-hash check and the decryption in one garage_ec_open_stripes call -- no CPU blake2 on this path.  A
    // block that does not hash to h, or that the configured stripe cannot serve (previous codes, replicas), goes
    // through rpc_get_block, with its stale-shard hunt, and the block it returns is opened.
    int rpc_get_block_opened(const Hash &h, const uint8_t *key, uint8_t *out, size_t cap, size_t *out_len)
    {
        Route route(*this);
        {
            SlotLease slot(grp().stripe_slots);
            uint8_t have[GARAGE_EC_MAX_K + GARAGE_EC_MAX_M];
            uint32_t block_len = 0;
            bool ok = false;
            gather_into(h, -1, slot.p, have, block_len, false, false, nullptr, &ok, nullptr, 0);
            if (ok) {
                const int rc = open_in_slot(h, key, slot.p, block_len, have, out, cap, out_len);
                if (rc != GARAGE_BM_E_CORRUPT_DATA) return rc;
            }
        }
        opened_fallbacks++;
        std::vector<uint8_t> blk(stored_max());
        size_t blen = 0;
        int rc = rpc_get_block(h, blk.data(), blk.size(), &blen);
        if (rc != GARAGE_BM_OK) return rc;
        SlotLease slot(grp().stripe_slots);
        uint8_t have[GARAGE_EC_MAX_K + GARAGE_EC_MAX_M] = {0};
        const size_t L = shard_len_of((uint32_t)blen);
        for (int j = 0; j < k; j++) {
            have[j] = 1;
            uint8_t *row = slot.p + (size_t)j * slot_stride;
            memset(row, 0, slot_stride);
            const size_t off = (size_t)j * L;
            if (off < blen) memcpy(row, blk.data() + off, std::min(L, blen - off));
        }
        return open_in_slot(h, key, slot.p, (uint32_t)blen, have, out, cap, out_len);
    }
    // PUT during a layout change: one shard per (node, index) request of garage_layout_write_plan, and the write quorum
    // in the node set of every active version (try_write_many_sets, rpc_helper.rs:432-538)
    int put_many_sets(const Layouts &ls, const Hash &h, uint32_t len, size_t L, const std::function<const uint8_t *(int)> &bytes,
                      const uint8_t *sums, int quorum)
    {
        const auto act = ls.raw();
        garage_shard_request reqs[(GARAGE_EC_MAX_K + GARAGE_EC_MAX_M) * GARAGE_BM_MAX_LAYOUT_VERSIONS];
        const int nr = garage_layout_write_plan(act.data(), (int)act.size(), h.data(), reqs, (int)(sizeof(reqs) / sizeof(reqs[0])));
        garage_quorum_tracker *t = nullptr;
        if (nr < 1 || garage_quorum_tracker_new(&t, reqs, nr, (int)act.size(), quorum) != GARAGE_LAYOUT_OK) return GARAGE_BM_E_MESSAGE;
        std::unique_ptr<garage_quorum_tracker, void (*)(garage_quorum_tracker *)> own(t, garage_quorum_tracker_free);
        for (int r = 0; r < nr; r++) {
            const int i = reqs[r].index;
            garage_quorum_tracker_register(t, r, write_shard(reqs[r].node, h, i, len, bytes(i), L, sums + (size_t)i * 32));
        }
        {
            std::lock_guard<std::mutex> lk(refs_mu);
            refs[h] = len;
        }
        return garage_quorum_tracker_state(t) == GARAGE_QUORUM_OK ? GARAGE_BM_OK : GARAGE_BM_E_QUORUM;
    }

    // manager.rs:344-363 + 276-339.  `out` must hold stored_max() bytes (a sealed block_size block); *out_len = the block's length.
    int rpc_get_block(const Hash &h, uint8_t *out, size_t cap, size_t *out_len)
    {
        Route route(*this);
        const int rc = get_from_stripe(h, out, cap, out_len, 0);
        if (rc == GARAGE_BM_OK || !has_legacy()) return rc;
        // the configured stripe cannot serve it (yet): a block stored before the code changed
        for (int c = 1; c < (int)codes.size(); c++)
            if (get_from_stripe(h, out, cap, out_len, c) == GARAGE_BM_OK) {
                legacy_gets++;
                return GARAGE_BM_OK;
            }
        uint32_t len = 0;
        if (read_replica(h, out, cap, len)) {
            *out_len = len;
            legacy_gets++;
            return GARAGE_BM_OK;
        }
        return rc;
    }

    // The gather of the ranged GETs.  The block length and tag kind come from the first configured-code shard header
    // that reads (a bad one quarantines its shard); pre(block_len) then returns 0 to go on, kRangeWhole or an error to
    // stop with.  plan (garage_ec_range_plan or garage_ec_open_range_plan) names the runs of range [off, off + len) to
    // fetch; each holder reads only the tag span covering its runs (garage_ec_tag_span) into `slot` and checks it against
    // the shard's tag; a span that fails, or a shard whose header does not match, quarantines its shard and the plan is
    // recomputed without it.  On GARAGE_BM_OK: `present` is the final plan's presence map, *gpu its needs_gpu, and
    // `fetched_ctr` has the planned run bytes added.  kRangeNoHeader if no configured-code header reads.
    static constexpr int kRangeWhole = 1, kRangeNoHeader = 2;
    using RangePlanFn = int (*)(const garage_ec_ctx *, const uint8_t *, uint32_t, uint32_t, uint32_t, garage_ec_range *,
                                size_t, size_t *, int *);
    int gather_ranged(const Hash &h, uint8_t *slot, const std::function<int(uint32_t)> &pre, RangePlanFn plan, uint32_t off,
                      uint32_t len, uint32_t &block_len, uint8_t *present, int *gpu, std::atomic<uint64_t> &read_ctr,
                      std::atomic<uint64_t> &fetched_ctr)
    {
        const Code &cd = codes[0];
        const int tot = cd.tot;
        ShardSources srcs = shard_sources(h, 0);
        ShardMeta m0;
        bool have_len = false;
        for (int i = 0; i < tot && !have_len; i++)
            for (; srcs.left(i); srcs.next(i)) {  // a down holder or a missing file: the next source
                ShardMeta mt;
                if (!read_shard_into(srcs.node(i), h, nullptr, 0, mt, false, 0, srcs.file(i), ShardSpan::bytes(0, 0)))
                    continue;
                if (mt.index == i) {
                    m0 = mt;
                    have_len = true;
                    break;
                }
                quarantine(srcs.node(i), h, 0, srcs.file(i));  // a misplaced shard
            }
        if (!have_len) return kRangeNoHeader;
        block_len = m0.block_len;
        const uint32_t L = (uint32_t)shard_len_of(block_len);
        int rc = pre(block_len);
        if (rc) return rc;
        uint8_t fetched[GARAGE_EC_MAX_K + GARAGE_EC_MAX_M] = {0};
        uint32_t f_lo[GARAGE_EC_MAX_K + GARAGE_EC_MAX_M], f_hi[GARAGE_EC_MAX_K + GARAGE_EC_MAX_M];
        std::vector<garage_ec_range> runs((size_t)tot * ((cd.clay ? cd.quantum / 16 : 1) + 2) * 2);
        size_t nr = 0;
        for (;;) {
            for (int i = 0; i < tot; i++) present[i] = fetched[i] || srcs.left(i);
            rc = plan(cd.ctx, present, block_len, off, len, runs.data(), runs.size(), &nr, gpu);
            if (rc == GARAGE_EC_E_UNRECOVERABLE) return GARAGE_BM_E_MISSING_BLOCK;
            if (rc != GARAGE_EC_OK) return rc;
            uint32_t lo[GARAGE_EC_MAX_K + GARAGE_EC_MAX_M], hi[GARAGE_EC_MAX_K + GARAGE_EC_MAX_M] = {0};
            for (int i = 0; i < tot; i++) lo[i] = UINT32_MAX;
            for (size_t x = 0; x < nr; x++) {
                lo[runs[x].shard] = std::min(lo[runs[x].shard], runs[x].offset);
                hi[runs[x].shard] = std::max(hi[runs[x].shard], runs[x].offset + runs[x].len);
            }
            bool replan = false;
            for (int i = 0; i < tot && !replan; i++) {
                if (lo[i] == UINT32_MAX || (fetched[i] && f_lo[i] <= lo[i] && hi[i] <= f_hi[i])) continue;
                uint32_t so = 0, sl = 0;
                if (garage_ec_tag_span(m0.sum_kind, L, lo[i], hi[i] - lo[i], &so, &sl) != GARAGE_EC_OK) return GARAGE_EC_E_INVALID;
                fetched[i] = 0;
                for (; srcs.left(i); srcs.next(i)) {  // a shard's runs come from one source
                    const int node = srcs.node(i), fidx = srcs.file(i);
                    ShardMeta mt;
                    bool got = read_shard_into(node, h, slot + (size_t)i * slot_stride + so, slot_stride - so, mt, true, 0,
                                               fidx, ShardSpan::bytes(so, sl));
                    if (got) read_ctr += sl;
                    if (got && (mt.index != i || mt.block_len != block_len || mt.shard_len != L)) {
                        quarantine(node, h, 0, fidx);  // a stale or misplaced shard with a self-consistent tag
                        got = false;
                    }
                    if (got) {
                        fetched[i] = 1;
                        f_lo[i] = so;
                        f_hi[i] = so + sl;
                        break;
                    }
                }
                replan = !fetched[i];  // the shard is out: the plan changes
            }
            if (!replan) break;
        }
        for (size_t x = 0; x < nr; x++) fetched_ctr += runs[x].len;
        return GARAGE_BM_OK;
    }

    // bytes [off, off + len) of the whole block (or plaintext) that `whole` -- rpc_get_block or rpc_get_block_opened --
    // writes into a stored_max() buffer: the ranged GETs' route through a whole-block GET
    int slice_whole(const std::function<int(uint8_t *, size_t, size_t *)> &whole, uint32_t off, uint32_t len, uint8_t *out,
                    size_t cap, size_t *out_len)
    {
        std::vector<uint8_t> buf(stored_max());
        size_t n = 0;
        const int rc = whole(buf.data(), buf.size(), &n);
        if (rc != GARAGE_BM_OK) return rc;
        if ((uint64_t)off + len > n || len > cap) return GARAGE_EC_E_INVALID;
        memcpy(out, buf.data() + off, len);
        *out_len = len;
        return GARAGE_BM_OK;
    }
    // a ranged item on the stripe gather_ranged left in `slot`, through the reconstruct dispatchers: a ranged GET, or
    // with a key a ranged opened GET
    int submit_range(uint8_t *slot, uint32_t block_len, const uint8_t *present, const uint8_t *key, uint32_t off,
                     uint32_t len, uint8_t *out)
    {
        ReconItem it;
        it.kind = key ? ReconItem::kOpenRange : ReconItem::kRange;
        it.stripe = slot;
        it.block_len = block_len;
        memcpy(it.present, present, tot);
        it.key = key;
        it.off = off;
        it.len = len;
        it.out = out;
        return grp().rec_batcher->submit(it);
    }

    // Bytes [off, off + len) of block h into out (S3 GetObject with a Range header, body_from_blocks_range; the
    // source ranges of UploadPartCopy), gathered by gather_ranged with garage_ec_range_plan.  A range whose touched data
    // shards are all present never touches the GPU; the others go through the reconstruct dispatchers
    // (garage_ec_decode_range_stripes).
    // Integrity: a ranged read is proven by the shard tags only.  The block's blake2sum needs the whole block, so a
    // self-consistent stale shard is found by the deep scrub (DESIGN.md section 5.4), not here.  A range equal to the
    // whole block is rpc_get_block, with its content-hash check and stale-shard hunt; so is a block held only under a
    // previous code or as replicas, which is then sliced.
    int rpc_get_block_range(const Hash &h, uint32_t off, uint32_t len, uint8_t *out, size_t cap, size_t *out_len)
    {
        Route route(*this);
        range_gets++;
        uint8_t present[GARAGE_EC_MAX_K + GARAGE_EC_MAX_M];
        uint32_t block_len = 0;
        int gpu = 0, rc;
        {
            SlotLease slot(grp().stripe_slots);
            rc = gather_ranged(
                h, slot.p,
                [&](uint32_t bl) -> int {
                    if ((uint64_t)off + len > bl || len > cap) return GARAGE_EC_E_INVALID;
                    return off == 0 && len == bl ? kRangeWhole : 0;
                },
                garage_ec_range_plan, off, len, block_len, present, &gpu, range_bytes_read, range_bytes_fetched);
            if (rc == GARAGE_BM_OK) {
                *out_len = len;
                if (!gpu) {  // every touched data shard is present: their range bytes, no GPU
                    const uint64_t L = shard_len_of(block_len);
                    for (uint64_t j = off / L, end = (uint64_t)off + len; j * L < end; j++) {
                        const uint64_t base = j * L, c0 = std::max<uint64_t>(off, base) - base,
                                       c1 = std::min<uint64_t>(end, base + L) - base;
                        memcpy(out + (base + c0 - off), slot.p + j * slot_stride + c0, c1 - c0);
                    }
                    return GARAGE_BM_OK;
                }
                range_degraded++;
                return submit_range(slot.p, block_len, present, nullptr, off, len, out);
            }
            if (rc == kRangeNoHeader && !has_legacy()) return GARAGE_BM_E_MISSING_BLOCK;
            if (rc != kRangeWhole && rc != kRangeNoHeader && !(rc == GARAGE_BM_E_MISSING_BLOCK && salvage_possible()))
                return rc;
        }
        const int r2 = slice_whole([&](uint8_t *b, size_t c, size_t *n) { return rpc_get_block(h, b, c, n); }, off, len, out,
                                   cap, out_len);
        // a range whose shards gave up: the whole GET's salvage (DESIGN.md section 5.14) serves it, else today's error
        return rc == GARAGE_BM_E_MISSING_BLOCK && r2 != GARAGE_BM_OK ? rc : r2;
    }

    // Plaintext bytes [off, off + len) of SSE-C block h sealed under key (a ranged GET or UploadPartCopy of an SSE-C
    // object, DESIGN.md sections 2.7 and 5.10), gathered by gather_ranged with garage_ec_open_range_plan: only the
    // nonce prefix and the chunks the range touches are fetched, and one garage_ec_open_range_stripes call of the
    // reconstruct dispatchers rebuilds, checks and decrypts them.  The whole plaintext, and blocks held only under a
    // previous code or as replicas, go through rpc_get_block_opened (content hash checked) and are sliced.  A touched
    // chunk that fails its tag is either a wrong key or a self-consistent stale shard, and at range level the two look
    // alike: one whole-block rpc_get_block_opened tells them apart (its hash check hunts and quarantines a stale
    // shard); its E_AUTH is the answer.
    int rpc_get_block_range_opened(const Hash &h, const uint8_t *key, uint32_t off, uint32_t len, uint8_t *out,
                                   size_t cap, size_t *out_len)
    {
        Route route(*this);
        struct Timer {
            std::atomic<uint64_t> &us;
            Clock::time_point t0;
            ~Timer() { us += us_since(t0); }
        } timer{sealed_range_us, Clock::now()};
        sealed_range_gets++;
        uint8_t present[GARAGE_EC_MAX_K + GARAGE_EC_MAX_M];
        uint32_t block_len = 0;
        int gpu = 0, rc;
        {
            SlotLease slot(grp().stripe_slots);
            rc = gather_ranged(
                h, slot.p,
                [&](uint32_t bl) -> int {
                    uint32_t P = 0;
                    if (!plain_len_of(bl, P)) return GARAGE_EC_E_AUTH;  // as garage_ec_sealed_range
                    if ((uint64_t)off + len > P || len > cap) return GARAGE_EC_E_INVALID;
                    return (off == 0 && len == P) || !len ? kRangeWhole : 0;
                },
                garage_ec_open_range_plan, off, len, block_len, present, &gpu, sealed_range_bytes_read,
                sealed_range_bytes_fetched);
            if (rc == GARAGE_BM_OK) {
                if (gpu) sealed_range_degraded++;
                rc = submit_range(slot.p, block_len, present, key, off, len, out);
                if (rc == GARAGE_BM_OK) *out_len = len;
            }
        }
        if (rc == kRangeWhole && !len) {  // a well-framed block's empty range
            *out_len = 0;
            return GARAGE_BM_OK;
        }
        if (rc == GARAGE_EC_E_AUTH || rc == kRangeWhole || (rc == kRangeNoHeader && has_legacy())) {
            if (rc == GARAGE_EC_E_AUTH) sealed_range_fallbacks++;
            rc = slice_whole([&](uint8_t *b, size_t c, size_t *n) { return rpc_get_block_opened(h, key, b, c, n); }, off, len,
                             out, cap, out_len);
            if (rc == GARAGE_EC_E_AUTH) sealed_range_auth_failures++;
            return rc;
        }
        return rc == kRangeNoHeader ? GARAGE_BM_E_MISSING_BLOCK : rc;
    }

    // the block from the first of its first legacy_rf ring nodes whose replica matches its content hash (a replica
    // that does not is quarantined)
    bool read_replica(const Hash &h, uint8_t *out, size_t cap, uint32_t &len, int *from = nullptr)
    {
        for (int i = 0; i < legacy_rf; i++) {
            const int node = ((int)h[0] % (int)nodes.size() + i) % (int)nodes.size();
            Node &nd = *nodes[node];
            ReadResult r;
            {
                std::lock_guard<std::mutex> lk(nd.mu);
                if (!nd.up) continue;
                r = nd.replica_read_into(h, out, cap, len);
            }
            if (r == kReadMissing) continue;
            Hash got;
            if (r == kReadOk) {
                bytes_read += len;
                garage_ec_blake2sum(out, len, got.data());
                if (got == h) {
                    if (from) *from = node;
                    return true;
                }
            }
            quarantine(node, h, -1);
        }
        return false;
    }

    // ---- salvage (DESIGN.md section 5.14) ------------------------------------------------------
    // Where the configured stripe has too few whole valid shards, an adler8 store can still hold every byte: each segment
    // of every index from the live shard or, failing that, from its quarantined copy, and each unit rebuilt on its own
    // (garage_ec_reconstruct_segments).  RS, LRC and PB stores with one active layout version only.
    bool salvage_possible() const { return sum_kind == GARAGE_EC_SUM_ADLER8 && !codes[0].clay && !multi_version(); }
    // the adler8 segment length of an L-byte shard
    static uint32_t seg_len(size_t L) { return (uint32_t)((L + 7) / 8 + 15) / 16 * 16; }
    // bit g: adler8 segment g of the L-byte shard b passes its value in the tag sum32 (an empty segment: set).  Salvage
    // and repair by segment keep a copy's segment on this proof alone.
    static uint8_t good_segments(const uint8_t *b, size_t L, const uint8_t *sum32)
    {
        const uint32_t S = seg_len(L);
        uint8_t bits = 0;
        for (uint32_t g = 0, o = 0; g < 8; g++, o += S)
            if (o >= L || garage_ec_check_shard_span_host(GARAGE_EC_SUM_ADLER8, b + o, (uint32_t)L, o,
                                                          (uint32_t)std::min<size_t>(S, L - o), sum32) == GARAGE_EC_OK)
                bits |= (uint8_t)(1u << g);
        return bits;
    }

    // The stripe of h rebuilt by segment into `slot` (a stripe slot) and proven by its content hash; the block goes to
    // blk (block_len bytes, nullable).  live_ok[i]: index i's live shard was whole and valid.  GARAGE_BM_OK, or
    // GARAGE_BM_E_MISSING_BLOCK when salvage does not apply or fails (never wrong bytes).
    int salvage_stripe(const Hash &h, uint8_t *slot, uint32_t &block_len, uint8_t *live_ok, uint8_t *blk = nullptr)
    {
        if (!salvage_possible()) return GARAGE_BM_E_MISSING_BLOCK;
        uint32_t expect = 0;
        {
            std::lock_guard<std::mutex> lk(refs_mu);
            auto it = refs.find(h);
            if (it == refs.end()) return GARAGE_BM_E_MISSING_BLOCK;
            expect = it->second;
        }
        salvage_attempts++;
        const size_t L = shard_len_of(expect);
        if (L > slot_stride) {
            salvage_failures++;
            return GARAGE_BM_E_MISSING_BLOCK;
        }
        const uint32_t S = seg_len(L);
        int who[64];
        storage_nodes_of(h, who);
        uint8_t seg[GARAGE_EC_MAX_K + GARAGE_EC_MAX_M];
        std::vector<uint8_t> tmp(slot_stride);
        uint64_t nread = 0, from_q = 0;
        // the header must name this index, the block length the others agree on (refs) and the adler8 tag
        auto fits = [&](const ShardMeta &mt, int i) {
            return mt.index == i && mt.block_len == expect && mt.shard_len == L && mt.sum_kind == GARAGE_EC_SUM_ADLER8;
        };
        for (int i = 0; i < tot; i++) {
            seg[i] = 0;
            live_ok[i] = 0;
            Node &nd = *nodes[who[i]];
            uint8_t *dst = slot + (size_t)i * slot_stride;
            for (int q = 0; q < 2 && seg[i] != 0xFF; q++) {  // the live copy first, then the quarantined one
                ShardMeta mt;
                ReadResult r;
                {
                    std::lock_guard<std::mutex> lk(nd.mu);
                    if (!nd.up) break;
                    r = nd.salvage_read(h, q == 1, q ? tmp.data() : dst, slot_stride, mt);
                }
                if (r != kReadOk || !fits(mt, i)) continue;
                nread += L;
                const uint8_t bits = (uint8_t)(good_segments(q ? tmp.data() : dst, L, mt.sum.data()) & ~seg[i]);
                if (q == 0) live_ok[i] = bits == 0xFF;
                for (uint32_t g = 0, o = 0; q && g < 8; g++, o += S)
                    if ((bits >> g) & 1 && o < L) {
                        memcpy(dst + o, tmp.data() + o, std::min<size_t>(S, L - o));
                        from_q++;
                    }
                seg[i] |= bits;
            }
        }
        salvage_bytes_read += nread;
        salvage_quarantined_segments += from_q;
        bool work = false;
        for (int i = 0; i < tot; i++) work |= seg[i] != 0xFF;
        if (work) {
            const uint32_t L32 = (uint32_t)L;
            int32_t st = 0;
            const auto t0 = Clock::now();
            const int rc = garage_ec_reconstruct_segments_stripes(grp().code_ctx[0], &slot, seg, nullptr, &st, &L32,
                                                                  slot_stride, 1);
            salvage_call_us += us_since(t0);
            if (rc != GARAGE_EC_OK || st != 0) {
                salvage_failures++;
                return GARAGE_BM_E_MISSING_BLOCK;
            }
            const bool pb = codes[0].pb;
            for (uint32_t g = 0; g < (pb ? 4u : 8u); g++)
                for (int i = 0; i < tot && (pb || (size_t)g * S < L); i++)
                    salvage_units_rebuilt += pb ? !((seg[i] >> g) & (seg[i] >> (g + 4)) & 1) : !((seg[i] >> g) & 1);
        }
        std::vector<uint8_t> own;
        if (!blk) {
            own.resize(expect);
            blk = own.data();
        }
        assemble(slot, expect, blk);
        if (!content_ok(h, blk, expect)) {  // e.g. a stale quarantined copy consistent with its own tag
            salvage_failures++;
            return GARAGE_BM_E_MISSING_BLOCK;
        }
        block_len = expect;
        salvage_blocks++;
        return GARAGE_BM_OK;
    }
    // A GET whose gather gave up: the salvaged block, or GARAGE_BM_E_MISSING_BLOCK as before.  Nothing is written: the
    // damaged indices were queued for resync when they were quarantined.
    int salvage_get(const Hash &h, uint8_t *slot, uint8_t *out, size_t cap, size_t *out_len)
    {
        uint8_t live[GARAGE_EC_MAX_K + GARAGE_EC_MAX_M];
        uint32_t bl = 0;
        std::vector<uint8_t> blk;
        {
            std::lock_guard<std::mutex> lk(refs_mu);
            auto it = refs.find(h);
            if (it == refs.end() || it->second > cap) return GARAGE_BM_E_MISSING_BLOCK;
        }
        if (salvage_stripe(h, slot, bl, live, out) != GARAGE_BM_OK) return GARAGE_BM_E_MISSING_BLOCK;
        *out_len = bl;
        return GARAGE_BM_OK;
    }
    // A resync or stripe repair whose survivors could not rebuild: salvage the stripe and write every shard whose live
    // copy was not whole and valid to its holder, with a fresh header and tag (.corrupted files stay).  Returns the shards
    // written (*bytes_out += their bytes); -1 if salvage failed; -2 if the write of index `must` failed.
    int salvage_heal(const Hash &h, uint8_t *slot, int must = -1, uint64_t *bytes_out = nullptr)
    {
        uint8_t live[GARAGE_EC_MAX_K + GARAGE_EC_MAX_M];
        uint32_t bl = 0;
        if (salvage_stripe(h, slot, bl, live) != GARAGE_BM_OK) return -1;
        int who[64];
        storage_nodes_of(h, who);
        const size_t L = shard_len_of(bl);
        int n = 0;
        bool must_ok = must < 0;
        for (int i = 0; i < tot; i++) {
            if (live[i]) continue;
            const uint8_t *bytes = slot + (size_t)i * slot_stride;
            Hash sum;
            shard_tag(bytes, L, sum);
            if (!write_shard(who[i], h, i, bl, bytes, L, sum.data())) continue;
            n++;
            if (bytes_out) *bytes_out += L;
            must_ok |= i == must;
        }
        return must_ok ? n : -2;
    }

    // ---- repair by segment (DESIGN.md section 5.15) -------------------------------------------
    // Resync of index idx of h on `node`, whose quarantined copy failed its adler8 tag (Node::tag_failed): the copy's
    // units that pass their segment tags stay, the others are rebuilt from the same columns of the survivors -- the
    // garage_ec_segment_read_ranges runs, each read through read_shard_into and checked against its holder's tag --
    // and the shard is written, with the copy's tag, only if all eight segment values match that tag.  `slot`: a
    // stripe slot.  true: written.  false: not tried (the store does not qualify, or the node holds no quarantined
    // copy) or failed (a fallback: a missing hint, a copy that does not fit, no good or no bad unit, an absent or bad
    // survivor span, an unrecoverable unit, a failed post-check or write); the caller rebuilds the whole shard.
    bool segment_repair(int node, const Hash &h, int idx, uint8_t *slot)
    {
        if (!salvage_possible()) return false;
        uint32_t expect = 0;
        {
            std::lock_guard<std::mutex> lk(refs_mu);
            auto it = refs.find(h);
            if (it == refs.end()) return false;
            expect = it->second;
        }
        const size_t L = shard_len_of(expect);
        Node &nd = *nodes[node];
        uint8_t *own = slot + (size_t)idx * slot_stride;
        ShardMeta cm;  // the copy's header
        ReadResult r = kReadMissing;
        {
            std::lock_guard<std::mutex> lk(nd.mu);
            if (!nd.up || !nd.has_quarantined(h)) return false;
            if (nd.tag_failed.count(h) && L <= slot_stride) r = nd.salvage_read(h, true, own, slot_stride, cm);
        }
        uint64_t nread = 0, fetched = 0, nshards = 0;
        auto count = [&] {
            segrep_bytes_read += nread;
            segrep_bytes_fetched += fetched;
            resync_bytes_read += nread;
            resync_bytes_fetched += fetched;
            resync_shards_read += nshards;
        };
        auto fallback = [&] {
            count();
            segrep_fallbacks++;
            return false;
        };
        if (r != kReadOk) return fallback();
        nread += L;
        if (cm.index != idx || cm.block_len != expect || cm.shard_len != L || cm.sum_kind != GARAGE_EC_SUM_ADLER8)
            return fallback();
        const bool pb = codes[0].pb;
        uint8_t bits = good_segments(own, L, cm.sum.data());
        if (pb) bits &= (uint8_t)((bits >> 4) | (bits << 4));  // a PB unit is segments g and g + 4: both or neither
        const uint32_t S = seg_len(L);
        int ngood = 0, nbad = 0;
        for (uint32_t g = 0; g < (pb ? 4u : 8u); g++)
            if (pb || (size_t)g * S < L) ((bits >> g) & 1 ? ngood : nbad)++;
        if (!ngood || !nbad) return fallback();
        // the survivors: every other index whose holder is up
        int who[64];
        storage_nodes_of(h, who);
        uint8_t seg[GARAGE_EC_MAX_K + GARAGE_EC_MAX_M], want[GARAGE_EC_MAX_K + GARAGE_EC_MAX_M] = {0};
        for (int i = 0; i < tot; i++) {
            Node &x = *nodes[who[i]];
            std::lock_guard<std::mutex> lk(x.mu);
            seg[i] = x.up ? 0xFF : 0x00;
        }
        seg[idx] = bits;
        want[idx] = 1;
        garage_ec_range runs[(GARAGE_EC_MAX_K + GARAGE_EC_MAX_M) * 8];
        size_t nr = 0;
        if (garage_ec_segment_read_ranges(codes[0].ctx, seg, want, (uint32_t)L, runs, sizeof(runs) / sizeof(runs[0]),
                                          &nr) != GARAGE_EC_OK)
            return fallback();
        for (size_t x = 0; x < nr; x++) {
            const garage_ec_range &rn = runs[x];
            ShardMeta mt;
            if (!read_shard_into(who[rn.shard], h, slot + (size_t)rn.shard * slot_stride + rn.offset,
                                 slot_stride - rn.offset, mt, /*for_dma=*/true, 0, -1, ShardSpan::bytes(rn.offset, rn.len)))
                return fallback();  // absent, or a span that failed its holder's tag (quarantined and queued)
            nread += rn.len;
            fetched += rn.len;
            nshards += x == 0 || runs[x - 1].shard != rn.shard;
            if (mt.index != (int)rn.shard || mt.block_len != expect || mt.shard_len != L) return fallback();
        }
        const uint32_t L32 = (uint32_t)L;
        int32_t st = 0;
        const auto t0 = Clock::now();
        const int rc = garage_ec_reconstruct_segments_stripes(grp().code_ctx[0], &slot, seg, want, &st, &L32, slot_stride, 1);
        segrep_call_us += us_since(t0);
        if (rc != GARAGE_EC_OK || st != 0) return fallback();
        Hash sum;
        shard_tag(own, L, sum);
        // the eight segment values written at PUT: a stale copy that rotted fails here
        if (memcmp(sum.data(), cm.sum.data(), 32) != 0) return fallback();
        if (!write_shard(node, h, idx, expect, own, L, cm.sum.data())) return fallback();
        count();
        segrep_repairs++;
        segrep_units_rebuilt += (uint64_t)nbad;
        resync_recv_counter++;
        resync_counter++;
        return true;
    }

    // manager.rs:344-363 + 276-339 on the stripe of `code`: gather, rebuild missing data shards, check the content
    // hash, and on a mismatch hunt the shard that is stale
    int get_from_stripe(const Hash &h, uint8_t *out, size_t cap, size_t *out_len, int code)
    {
        const int k = codes[code].k;
        SlotLease slot(grp().stripe_slots);
        uint8_t have[GARAGE_EC_MAX_K + GARAGE_EC_MAX_M], want[GARAGE_EC_MAX_K + GARAGE_EC_MAX_M] = {0};
        uint32_t block_len = 0;
        bool ok = false;
        gather_into(h, -1, slot.p, have, block_len, false, false, nullptr, &ok, nullptr, code);
        if (!ok)  // manager.rs:336-338, unless the stripe can be salvaged segment by segment
            return code == 0 ? salvage_get(h, slot.p, out, cap, out_len) : GARAGE_BM_E_MISSING_BLOCK;
        *out_len = block_len;
        if (block_len > cap) return GARAGE_EC_E_INVALID;
        bool all_data = true;
        for (int j = 0; j < k; j++) {
            all_data &= have[j] != 0;
            want[j] = !have[j];
        }
        if (!all_data) {
            int rc = reconstruct_in_slot(slot.p, block_len, have, want, code);
            if (rc != GARAGE_BM_OK) return rc;
        }
        assemble(slot.p, block_len, out, code);
        if (content_ok(h, out, block_len)) return GARAGE_BM_OK;
        return hunt_stale_shard(h, slot.p, out, cap, out_len, code);
    }

    // Every shard passed its own tag, yet the block is not the one `h` names: some shard is
    // stale or was rebuilt wrongly.  Find it: gather everything (into the stripe slot `sp`), drop one shard at a
    // time, rebuild, re-check (manager.rs read path: CorruptData -> quarantine + resync).
    int hunt_stale_shard(const Hash &h, uint8_t *sp, uint8_t *out, size_t cap, size_t *out_len, int code)
    {
        const int k = codes[code].k, tot = codes[code].tot;
        uint8_t have[GARAGE_EC_MAX_K + GARAGE_EC_MAX_M];
        uint32_t block_len = 0;
        corrupt_data_errors++;
        int who[GARAGE_EC_MAX_K + GARAGE_EC_MAX_M];
        const int avail = gather_into(h, -1, sp, have, block_len, /*all=*/true, /*for_gpu=*/true, nullptr, nullptr,
                                      nullptr, code, who);
        if (avail > k && block_len <= cap) {
            SlotLease trial(grp().stripe_slots);
            for (int x = 0; x < tot; x++) {
                if (!have[x]) continue;
                uint8_t h2[GARAGE_EC_MAX_K + GARAGE_EC_MAX_M], w2[GARAGE_EC_MAX_K + GARAGE_EC_MAX_M] = {0};
                memcpy(h2, have, tot);
                h2[x] = 0;
                bool need = false;
                for (int j = 0; j < k; j++) {
                    w2[j] = !h2[j];
                    need |= w2[j] != 0;
                }
                memcpy(trial.p, sp, (size_t)tot * slot_stride);
                if (need && reconstruct_in_slot(trial.p, block_len, h2, w2, code) != GARAGE_BM_OK) continue;
                assemble(trial.p, block_len, out, code);
                if (content_ok(h, out, block_len)) {
                    quarantine(who[x], h, code, code == 0 && multi_version() ? x : -1);  // the culprit
                    *out_len = block_len;
                    return GARAGE_BM_OK;
                }
            }
        }
        return GARAGE_BM_E_CORRUPT_DATA;
    }

    bool deletable_now(const Hash &h)  // refs_mu held.  rc.is_deletable() + BLOCK_GC_DELAY (rc.rs, manager.rs:49-52)
    {
        auto it = rc.find(h);
        if (it == rc.end() || it->second.count > 0) return false;
        return Clock::now() - it->second.zero_since >= std::chrono::milliseconds(cfg.block_gc_delay_ms);
    }

    // refs_mu held: ms until h, at rc 0, leaves its GC delay (at least 1)
    int64_t gc_delay_left_ms(const Hash &h)
    {
        const auto it = rc.find(h);
        const auto left = std::chrono::milliseconds(cfg.block_gc_delay_ms) - (Clock::now() - it->second.zero_since);
        return std::max<int64_t>(1, std::chrono::ceil<std::chrono::milliseconds>(left).count());
    }

    // gc_wait_ms: a block still inside its GC delay is not queued again; *gc_wait_ms = the ms until it leaves it (0 if
    // it is not such a block)
    int resync_block(int node, const Hash &h, int64_t *gc_wait_ms = nullptr)
    {
        Route route(*this);
        if (gc_wait_ms) *gc_wait_ms = 0;
        const auto ls = layouts();
        const bool multi = ls->v.size() > 1;
        const int idx = newest_index(h, node);
        if (idx < 0) return GARAGE_BM_OK;  // not a storage node for it any more (resync.rs:466-477)
        bool known, unneeded;
        {
            // the deletion decision and the deletion itself happen under BOTH locks (refs_mu, then the
            // node's): an incref / re-PUT cannot slip in between the check and the erase
            std::lock_guard<std::mutex> rl(refs_mu);
            known = refs.count(h) != 0;
            auto it = rc.find(h);
            unneeded = it != rc.end() && it->second.count <= 0;
            Node &nd = *nodes[node];
            std::lock_guard<std::mutex> lk(nd.mu);
            if (!nd.up) return GARAGE_BM_E_MESSAGE;
            const bool exists = nd.store_has(h, multi ? idx : -1);
            // during a layout change the node's files of every index go, an older index moved aside included
            const bool held = multi && !nd.other_index_files(h, -1).empty();
            if ((exists || held) && unneeded) {  // offload branch, resync.rs:369-458: delete_if_unneeded
                if (!deletable_now(h)) {  // still inside the GC delay: look again later
                    if (gc_wait_ms) *gc_wait_ms = gc_delay_left_ms(h);
                    else nd.schedule(h, now_ms());
                    return GARAGE_BM_OK;
                }
                delete_counter += multi ? nd.erase_other_indices(h, -1, [] { return true; }) : nd.store_erase(h);
                return GARAGE_BM_OK;
            }
            if (exists) return GARAGE_BM_OK;
        }
        if (!known || unneeded) return GARAGE_BM_OK;  // rc == 0: nothing to fetch
        SlotLease slot(grp().stripe_slots);
        if (multi) {  // a layout change: the shard's holder in an older version is asked first (DESIGN.md section 5.2)
            const int c = copy_from_older(node, h, idx, *ls, false, slot.p);
            if (c != 0) {
                (c > 0 ? resync_counter : resync_error_counter)++;
                return c > 0 ? GARAGE_BM_OK : GARAGE_BM_E_MESSAGE;
            }
        }
        // a shard whose tag failed: only its damaged units, from the same columns of the survivors (DESIGN.md 5.15)
        if (segment_repair(node, h, idx, slot.p)) return GARAGE_BM_OK;
        uint8_t have[GARAGE_EC_MAX_K + GARAGE_EC_MAX_M], want[GARAGE_EC_MAX_K + GARAGE_EC_MAX_M] = {0};
        uint32_t block_len = 0;
        bool ok = false;
        want[idx] = 1;
        uint64_t nbytes = 0;
        resync_shards_read += (uint64_t)gather_into(h, node, slot.p, have, block_len, false, /*for_gpu=*/true, want, &ok,
                                                    &nbytes);
        const uint64_t fetched = ok ? fetched_bytes(have, want, block_len, nbytes) : nbytes;
        resync_bytes_read += nbytes;
        resync_bytes_fetched += fetched;
        if (multi) {
            layout_bytes_read += nbytes;
            layout_bytes_fetched += fetched;
        }
        if (!ok) {
            // no configured stripe to rebuild from, but maybe a block stored before the code changed: convert it
            if (has_legacy() && convert_batch({h}) == 1) {
                resync_counter++;
                return GARAGE_BM_OK;
            }
            // rebuild by segment from the survivors and the quarantined copies (DESIGN.md section 5.14)
            if (salvage_possible()) {
                const int w = salvage_heal(h, slot.p, idx);
                if (w >= 0) {
                    resync_counter++;
                    return GARAGE_BM_OK;
                }
                if (w == -2) {
                    resync_error_counter++;
                    return GARAGE_BM_E_MESSAGE;  // as a failed write of the fetch branch
                }
            }
            resync_error_counter++;
            resync_failed_bytes_read += nbytes;
            return GARAGE_BM_E_MISSING_BLOCK;  // resync.rs:488-494
        }
        int rc2 = reconstruct_in_slot(slot.p, block_len, have, want);
        if (rc2 != GARAGE_BM_OK) {
            resync_error_counter++;
            resync_failed_bytes_read += nbytes;
            return rc2;
        }
        resync_recv_counter++;
        const size_t L = shard_len_of(block_len);
        const uint8_t *bytes = slot.p + (size_t)idx * slot_stride;
        Hash sum;
        shard_tag(bytes, L, sum);
        if (!write_shard(node, h, idx, block_len, bytes, L, sum.data())) {  // resync.rs:499
            resync_error_counter++;
            resync_failed_bytes_read += nbytes;
            return GARAGE_BM_E_MESSAGE;  // Error::Io: stays queued, the caller backs off (resync.rs:300-315)
        }
        if (multi) {
            layout_shards_rebuilt++;
            layout_bytes_written += L;
        }
        resync_counter++;
        return GARAGE_BM_OK;
    }

    // ---- changing the cluster layout (DESIGN.md section 5.2) ---------------------------------
    // Receive, first choice: shard idx of h, which the newest version gives `node`, copied from the node that holds idx
    // in an older active version (oldest first), its tag and header checked on read and kept.  1: copied; 0: no valid
    // copy (rebuild it); -1: the write to `node` failed.  `buf`: slot_stride bytes.
    int copy_from_older(int node, const Hash &h, int idx, const Layouts &ls, bool counted, uint8_t *buf)
    {
        uint32_t expect = 0;
        bool have_expect = false;
        {
            std::lock_guard<std::mutex> lk(refs_mu);
            auto it = refs.find(h);
            if (it != refs.end()) expect = it->second, have_expect = true;
        }
        for (size_t v = 0; v + 1 < ls.v.size(); v++) {
            int32_t row[GARAGE_EC_MAX_K + GARAGE_EC_MAX_M];
            garage_layout_nodes_of(ls.v[v].get(), h.data(), row);
            const int y = row[idx];
            ShardMeta mt;
            if (y == node || !read_shard_into(y, h, buf, slot_stride, mt, false, 0, idx)) continue;
            layout_bytes_read += mt.shard_len;
            layout_bytes_fetched += mt.shard_len;
            if (mt.index != idx || (have_expect && mt.block_len != expect)) {
                quarantine(y, h, 0, idx);  // a self-consistent shard of another block length: stale
                continue;
            }
            if (!write_shard(node, h, idx, mt.block_len, buf, mt.shard_len, mt.sum.data(), counted)) return -1;
            layout_shards_copied++;
            layout_bytes_written += mt.shard_len;
            return 1;
        }
        return 0;
    }
    // One stripe of a rebuild batch: the shards `want` of h are rebuilt and shard i is written to node to[i].  skip: a
    // node whose wanted shards are not read (a layout sync's receiver), -1 none.  grow: a survivor the gather
    // quarantines becomes one more wanted shard if its holder to[i] is up, and the stripe is gathered again for it.
    struct RebuildJob {
        Hash h{};
        uint8_t want[GARAGE_EC_MAX_K + GARAGE_EC_MAX_M] = {0};
        int to[GARAGE_EC_MAX_K + GARAGE_EC_MAX_M] = {0};
        int skip = -1;
        bool grow = false;
        int written = 0;  // out: the shards written; -1: the stripe could not be rebuilt
    };
    // where a rebuild batch counts: the bytes read and handed to the rebuild, the shards and bytes written, the errors
    // (an unrecoverable stripe, a failed write: one each) and the time of its reconstruct calls (nullable)
    struct RebuildCounters {
        std::atomic<uint64_t> &read, &fetched, &shards, &written, &errors;
        std::atomic<uint64_t> *call_us;
        bool counted;  // the writes are file operations of garage_bm_debug_convert_stop_after
    };
    // Rebuild the jobs' stripes from their survivors, like resync_block's fetch branch, batch_max_blocks stripes per
    // garage_ec_reconstruct_stripes.  Returns the number of shards written; *errors = the errors counted.
    // Concurrent callers run their batches one at a time (rebuild_mu), and a batch takes its stripe slots from the
    // group's pool in one step, so it never holds part of the pool while it waits for the rest.
    size_t rebuild_batch(std::vector<RebuildJob> &jobs, const RebuildCounters &c, size_t *errors = nullptr)
    {
        DeviceGroup &dg = grp();
        std::lock_guard<std::mutex> rl(dg.rebuild_mu);
        const size_t bmax = std::max<uint32_t>(cfg.batch_max_blocks, 1);
        std::atomic<size_t> written{0}, nerr{0};
        for (size_t b0 = 0; b0 < jobs.size(); b0 += bmax) {
            const size_t n = std::min(bmax, jobs.size() - b0);
            struct Slots {
                SlotPool &pool;
                std::vector<uint8_t *> p;
                ~Slots() { pool.release_n(p); }
            } slots{dg.stripe_slots, dg.stripe_slots.acquire_n(n)};
            std::vector<ReconItem> items(n);
            std::vector<uint8_t> ok(n, 0);
            parallel_for(n, [&](size_t j, std::vector<uint8_t> &) {
                const RebuildJob &jb = jobs[b0 + j];
                ReconItem &it = items[j];
                it.stripe = slots.p[j];
                it.call_us = c.call_us;
                memcpy(it.want, jb.want, tot);
                for (;;) {
                    bool g = false;
                    uint64_t nbytes = 0;
                    gather_into(jb.h, jb.skip, it.stripe, it.present, it.block_len, false, /*for_gpu=*/true, it.want, &g,
                                &nbytes);
                    c.read += nbytes;
                    c.fetched += g ? fetched_bytes(it.present, it.want, it.block_len, nbytes) : nbytes;
                    ok[j] = g;
                    bool more = false;
                    for (int i = 0; jb.grow && i < tot; i++)
                        if (!it.want[i] && !it.present[i] && probe(jb.to[i], jb.h, i) == 0) {
                            it.want[i] = 1;
                            more = true;
                        }
                    if (!more) break;
                }
            });
            std::vector<ReconItem *> batch;
            for (size_t j = 0; j < n; j++)
                if (ok[j]) batch.push_back(&items[j]);
            std::vector<int> rc;
            reconstruct_calls += batch.size();
            if (!batch.empty()) dg.rec_batcher->submit_all(batch, rc);
            for (size_t q = 0, j = 0; j < n; j++)
                if (ok[j]) ok[j] = rc[q++] == GARAGE_BM_OK;
            parallel_for(n, [&](size_t j, std::vector<uint8_t> &) {
                RebuildJob &jb = jobs[b0 + j];
                if (!ok[j]) {
                    jb.written = -1;
                    c.errors++;
                    nerr++;
                    return;
                }
                const uint32_t len = items[j].block_len;
                const size_t L = shard_len_of(len);
                for (int i = 0; i < tot; i++) {
                    if (!items[j].want[i]) continue;
                    const uint8_t *bytes = items[j].stripe + (size_t)i * slot_stride;
                    Hash sum;
                    shard_tag(bytes, L, sum);
                    if (!write_shard(jb.to[i], jb.h, i, len, bytes, L, sum.data(), c.counted)) {
                        c.errors++;
                        nerr++;
                        continue;
                    }
                    c.shards++;
                    c.written += L;
                    jb.written++;
                    written++;
                }
            });
        }
        if (errors) *errors = nerr;
        return written;
    }
    // what holder `node` says of shard i of h: 1 it holds a valid-looking one (Node::store_probe), 0 it does not, -1 down
    int probe(int node, const Hash &h, int i)
    {
        Node &nd = *nodes[node];
        std::lock_guard<std::mutex> lk(nd.mu);
        if (!nd.up) return -1;
        return nd.store_probe(h, i) ? 1 : 0;
    }
    // the newest version's stripe of h holds its write quorum: k+1 configured-code shards with valid tags on their nodes.
    // by_index: each read from the file holding its assigned index (the newest stripe during a layout change)
    bool at_quorum(const Hash &h, uint8_t *buf, bool by_index)
    {
        int who[64];
        storage_nodes_of(h, who);
        const int quorum = garage_ec_write_quorum(k, m, GARAGE_CONSISTENT);
        int good = 0;
        for (int i = 0; i < tot && good < quorum && good + (tot - i) >= quorum; i++) {
            ShardMeta mt;
            if (read_shard_into(who[i], h, buf, slot_stride, mt, false, 0, by_index ? i : -1) && mt.index == i) good++;
        }
        return good >= quorum;
    }
    // Offload of shard i of h from `node` (resync.rs:369-458): the newest version's holder of i gets it first if it
    // lacks it (a push: the copy a receiver would make), then the file goes once the newest stripe holds k+1.
    // Returns the number of shards pushed.
    int offload_shards(int node, const Hash &h, uint8_t *buf)
    {
        Node &nd = *nodes[node];
        int who[64];
        storage_nodes_of(h, who);
        const int a = newest_index(h, node);
        std::vector<std::pair<const char *, int>> held;
        {
            std::lock_guard<std::mutex> lk(nd.mu);
            held = nd.other_index_files(h, a);
        }
        int pushed = 0;
        bool all_held = true;  // every newest holder of an index this node offloads has it
        for (auto &f : held) {
            const int i = f.second;
            ShardMeta mt;
            if (read_shard_into(who[i], h, buf, slot_stride, mt, false, 0, i) && mt.index == i) continue;
            if (read_shard_into(node, h, buf, slot_stride, mt, false, 0, i) && mt.index == i &&
                write_shard(who[i], h, i, mt.block_len, buf, mt.shard_len, mt.sum.data(), true)) {
                layout_shards_copied++;
                layout_bytes_read += mt.shard_len;
                layout_bytes_fetched += mt.shard_len;
                layout_bytes_written += mt.shard_len;
                pushed++;
            } else {
                all_held = false;
            }
        }
        if (held.empty() || !all_held || !at_quorum(h, buf, true)) return pushed;
        std::lock_guard<std::mutex> lk(nd.mu);
        if (nd.up) layout_deleted += nd.erase_other_indices(h, a, [this] { return convert_op_allowed(); });
        return pushed;
    }
    // garage_bm_layout_sync_step: see include/garage_block_manager.h
    int layout_sync_step(int node, const Hash *cursor, size_t max_blocks, Hash *cursor_out, int *finished, uint64_t *moved)
    {
        Route route(*this);
        Node &nd = *nodes[node];
        const auto ls = layouts();
        const uint64_t newest_v = garage_layout_version(ls->newest());
        std::vector<Hash> hs;
        {
            std::lock_guard<std::mutex> lk(refs_mu);
            for (auto &kv : refs) hs.push_back(kv.first);
        }
        hs.erase(std::remove_if(hs.begin(), hs.end(), [&](const Hash &h) { return newest_index(h, node) < 0; }), hs.end());
        {
            std::lock_guard<std::mutex> lk(nd.mu);
            if (!nd.up) return GARAGE_BM_E_MESSAGE;
            if (!nd.dir.empty()) nd.store_list(hs);
        }
        int done = 0;
        sweep_page(hs, cursor, max_blocks, cursor_out, &done);
        if (finished) *finished = done;
        if (!cursor) {
            std::lock_guard<std::mutex> lk(layout_mu);
            pass_version[node] = newest_v;
            pass_clean[node] = 1;
        }
        std::vector<std::pair<Hash, int>> receive;
        std::vector<Hash> offload;  // blocks of which the node holds an index the newest version does not give it
        {
            SlotLease scratch(grp().stripe_slots);
            for (const Hash &h : hs) {
                {
                    // rc 0: nothing is received; the node's shards go once the GC delay has passed, decided and deleted
                    // under both locks like resync_block's offload branch
                    std::lock_guard<std::mutex> rl(refs_mu);
                    auto it = rc.find(h);
                    if (it != rc.end() && it->second.count <= 0) {
                        if (deletable_now(h)) {
                            std::lock_guard<std::mutex> lk(nd.mu);
                            delete_counter += nd.erase_other_indices(h, -1, [this] { return convert_op_allowed(); });
                        }
                        continue;
                    }
                    if (!refs.count(h)) continue;  // a file of no known block
                }
                const int a = newest_index(h, node);
                ShardMeta mt;
                if (a >= 0 && !(read_shard_into(node, h, scratch.p, slot_stride, mt, false, 0, a) && mt.index == a))
                    receive.emplace_back(h, a);
                std::lock_guard<std::mutex> lk(nd.mu);
                if (!nd.other_index_files(h, a).empty()) offload.push_back(h);
            }
        }
        std::atomic<bool> clean{true};
        std::atomic<uint64_t> n_moved{0};
        std::vector<std::pair<Hash, int>> rebuild;
        std::mutex rebuild_mu;
        parallel_for(receive.size(), [&](size_t j, std::vector<uint8_t> &buf) {
            buf.resize(slot_stride);
            const int c = copy_from_older(node, receive[j].first, receive[j].second, *ls, true, buf.data());
            if (c > 0) {
                n_moved++;
            } else if (c == 0) {
                std::lock_guard<std::mutex> lk(rebuild_mu);
                rebuild.push_back(receive[j]);
            } else {
                layout_sync_errors++;
                clean = false;
            }
        });
        std::sort(rebuild.begin(), rebuild.end());
        std::vector<RebuildJob> jobs(rebuild.size());
        for (size_t j = 0; j < rebuild.size(); j++) {
            jobs[j].h = rebuild[j].first;
            jobs[j].want[rebuild[j].second] = 1;
            jobs[j].to[rebuild[j].second] = node;
            jobs[j].skip = node;
        }
        size_t errs = 0;
        n_moved += rebuild_batch(jobs, {layout_bytes_read, layout_bytes_fetched, layout_shards_rebuilt, layout_bytes_written,
                                        layout_sync_errors, nullptr, true},
                                 &errs);
        if (errs) clean = false;
        // offload: deleted only once the newest stripe is seen at its write quorum (the deletion rule of DESIGN.md 5.1)
        parallel_for(offload.size(), [&](size_t j, std::vector<uint8_t> &buf) {
            buf.resize(slot_stride);
            n_moved += offload_shards(node, offload[j], buf.data());
        });
        if (moved) *moved = n_moved;
        std::lock_guard<std::mutex> lk(layout_mu);
        if (!clean) pass_clean[node] = 0;
        if (done && pass_clean[node] && pass_version[node] == newest_v && synced[node] < newest_v) {
            synced[node] = newest_v;
            retire_if_synced();
            if (layout_file && !save_layout(*layouts())) return GARAGE_BM_E_MESSAGE;
        }
        return GARAGE_BM_OK;
    }
    // layout_mu held: once every storage node of the newest version has synced it, the older versions are dropped
    void retire_if_synced()
    {
        const auto ls = layouts();
        if (ls->v.size() < 2) return;
        const uint64_t newest_v = garage_layout_version(ls->newest());
        const auto &cap = ls->capacity.back();
        for (size_t n = 0; n < nodes.size(); n++)
            if (cap[n] > 0 && synced[n] < newest_v) return;
        auto nl = std::make_shared<Layouts>();
        nl->v.push_back(ls->v.back());
        nl->zone.push_back(ls->zone.back());
        nl->capacity.push_back(ls->capacity.back());
        std::atomic_store(&layouts_, std::shared_ptr<const Layouts>(std::move(nl)));
    }
    // The layout history, <data_dir>/layout (Garage keeps its cluster layout in metadata, not in its config): every
    // active version's spec and ring, and each node's synced version.  tmp -> fsync -> rename, then the directory
    // under data_fsync.  layout_mu held (or the manager not yet shared).
    std::string layout_path;
    bool save_layout(const Layouts &ls)
    {
        std::string s = "garage-bm-layout 1\nnodes " + std::to_string(nodes.size()) + " shards " + std::to_string(tot) + "\n";
        std::vector<uint8_t> ring((size_t)GARAGE_NB_PARTITIONS * tot);
        for (size_t v = 0; v < ls.v.size(); v++) {
            s += "version " + std::to_string(garage_layout_version(ls.v[v].get())) + "\nzone";
            for (int32_t z : ls.zone[v]) s += " " + std::to_string(z);
            s += "\ncapacity";
            for (uint64_t c : ls.capacity[v]) s += " " + std::to_string(c);
            garage_layout_ring(ls.v[v].get(), ring.data());
            s += "\nring " + hex_of(ring.data(), ring.size()) + "\n";
        }
        s += "synced";
        for (uint64_t v : synced) s += " " + std::to_string(v);
        s += "\n";
        return write_file_atomic(layout_path, s.data(), s.size(), nullptr, 0, true, cfg.data_fsync != 0);
    }
    // 1: loaded into out / syn; 0: no file; -1: a file this manager cannot use
    static int load_layout(const std::string &path, int n, int tot, Layouts &out, std::vector<uint64_t> &syn)
    {
        std::string s;
        if (!read_file(path, s)) return 0;
        std::vector<std::string> tok;  // whitespace-separated words
        for (size_t i = 0; i < s.size();) {
            while (i < s.size() && isspace((unsigned char)s[i])) i++;
            const size_t j = i;
            while (i < s.size() && !isspace((unsigned char)s[i])) i++;
            if (i > j) tok.push_back(s.substr(j, i - j));
        }
        size_t t = 0;
        auto word = [&](const char *w) { return t < tok.size() && tok[t] == w ? (t++, true) : false; };
        auto num = [&](auto &v) {
            if (t >= tok.size()) return false;
            char *e = nullptr;
            errno = 0;
            const long long x = strtoll(tok[t].c_str(), &e, 10);
            if (errno || *e || tok[t].empty()) return false;
            v = (std::remove_reference_t<decltype(v)>)x;
            t++;
            return true;
        };
        int fmt = 0, fn = 0, ft = 0;
        if (!word("garage-bm-layout") || !num(fmt) || fmt != 1) return -1;
        if (!word("nodes") || !num(fn) || !word("shards") || !num(ft) || fn != n || ft != tot) return -1;
        while (word("version")) {
            uint64_t v = 0;
            std::vector<int32_t> zone(n);
            std::vector<uint64_t> cap(n);
            if (!num(v) || !word("zone")) return -1;
            for (auto &z : zone)
                if (!num(z)) return -1;
            if (!word("capacity")) return -1;
            for (auto &c : cap)
                if (!num(c)) return -1;
            if (!word("ring") || t >= tok.size() || tok[t].size() != (size_t)GARAGE_NB_PARTITIONS * tot * 2) return -1;
            const std::string &hex = tok[t++];
            std::vector<uint8_t> ring(hex.size() / 2);
            for (size_t i = 0; i < ring.size(); i++) {
                char *e = nullptr;
                const std::string b = hex.substr(2 * i, 2);
                ring[i] = (uint8_t)strtoul(b.c_str(), &e, 16);
                if (*e) return -1;
            }
            garage_layout *l = nullptr;
            if (garage_layout_from_ring(&l, v, n, zone.data(), cap.data(), tot, ring.data()) != GARAGE_LAYOUT_OK) return -1;
            out.v.emplace_back(l, garage_layout_free);
            out.zone.push_back(std::move(zone));
            out.capacity.push_back(std::move(cap));
        }
        if (!word("synced") || out.v.empty() || out.v.size() > GARAGE_BM_MAX_LAYOUT_VERSIONS) return -1;
        syn.assign(n, 0);
        for (auto &v : syn)
            if (!num(v)) return -1;
        return 1;
    }
    // garage_bm_apply_layout: see include/garage_block_manager.h
    int apply_layout(const garage_bm_layout_spec *spec, uint64_t *version_out)
    {
        if (nodes[0]->dir.empty() || has_legacy() || (codes[0].clay && !cfg.clay_layout)) return GARAGE_EC_E_INVALID;
        std::lock_guard<std::mutex> lk(layout_mu);
        const auto ls = layouts();
        if (!ls->newest() || ls->v.size() >= GARAGE_BM_MAX_LAYOUT_VERSIONS) return GARAGE_EC_E_INVALID;
        const uint64_t v = garage_layout_version(ls->newest()) + 1;
        auto nl = std::make_shared<Layouts>(*ls);
        if (!layout_from_spec(*nl, v, (int)nodes.size(), k, m, spec, ls->newest())) return GARAGE_EC_E_INVALID;
        if (!save_layout(*nl)) return GARAGE_BM_E_MESSAGE;  // on disk before any shard goes to the new version
        for (auto &nd : nodes) nd->by_index = true;           // from now on a node may hold two indices of a block
        layout_file = true;
        std::atomic_store(&layouts_, std::shared_ptr<const Layouts>(std::move(nl)));
        if (version_out) *version_out = v;
        return GARAGE_BM_OK;
    }
    // a spec's layout version appended to `out`; false for a spec garage_bm_config.layout documents as invalid
    static bool layout_from_spec(Layouts &out, uint64_t version, int n, int k, int m, const garage_bm_layout_spec *s,
                                 const garage_layout *previous)
    {
        if (!s || !s->zone || !s->capacity || s->zone_redundancy < 0 || s->max_per_zone < 0 || s->max_per_zone > m ||
            n > GARAGE_LAYOUT_MAX_NODES)
            return false;
        int storage = 0;
        for (int i = 0; i < n; i++) storage += s->capacity[i] > 0;
        if (storage < k + m) return false;
        garage_layout *l = nullptr;
        if (garage_layout_compute(&l, version, n, s->zone, s->capacity, k + m, s->zone_redundancy, s->max_per_zone, previous) !=
            GARAGE_LAYOUT_OK)
            return false;
        out.v.emplace_back(l, garage_layout_free);
        out.zone.emplace_back(s->zone, s->zone + n);
        out.capacity.emplace_back(s->capacity, s->capacity + n);
        return true;
    }

    // ---- changing the store's code (DESIGN.md section 5.1) ----------------------------------
    // every node that may hold a legacy copy of a block is among the first legacy_row() nodes of its ring row
    int legacy_row() const
    {
        int r = legacy_rf;
        for (size_t c = 1; c < codes.size(); c++) r = std::max(r, codes[c].tot);
        return r;
    }
    // the node that converts h: the first up node holding a legacy copy, previous codes in order and their shards in
    // index order, then the replica holders; -1 if no up node holds one
    int converter_of(const Hash &h)
    {
        for (int c = 1; c < (int)codes.size(); c++)
            for (int i = 0; i < codes[c].tot; i++) {
                Node &nd = *nodes[ring_node(h, i)];
                std::lock_guard<std::mutex> lk(nd.mu);
                if (nd.up && nd.has_code(h, c)) return ring_node(h, i);
            }
        for (int i = 0; i < legacy_rf; i++) {
            Node &nd = *nodes[ring_node(h, i)];
            std::lock_guard<std::mutex> lk(nd.mu);
            if (nd.up && nd.has_replica(h)) return ring_node(h, i);
        }
        return -1;
    }
    // node's legacy copies of h are removed, each removal one conversion file operation.  Only called once the
    // caller has seen the configured stripe at quorum, or for a block whose rc is 0 (then with refs_mu held).
    void delete_legacy(int node, const Hash &h)
    {
        Node &nd = *nodes[node];
        std::lock_guard<std::mutex> lk(nd.mu);
        if (nd.up && !nd.dir.empty()) legacy_deleted += nd.store_erase_legacy(h, [this] { return convert_op_allowed(); });
    }
    // Rewrite blocks stored under a previous code or as replicas under the configured code: one garage_ec_transcode
    // per source (previous codes in order, then replicas) and batch of batch_max_blocks.  Nothing is written for a
    // block whose new data shards do not hash to it; then the old stripe's stale shard is hunted and quarantined and
    // the block converted from the consistent rest.  A block is converted once k+1 new shards are durable; then the
    // legacy copies on the up nodes are deleted.  Returns the number converted; a block that fails keeps every legacy
    // copy and counts in convert_errors.
    size_t convert_batch(const std::vector<Hash> &hs)
    {
        std::lock_guard<std::mutex> cl(convert_mu);
        DeviceGroup &dg = grp();
        const size_t bmax = std::max<uint32_t>(cfg.batch_max_blocks, 1);
        const int nsrc = (int)codes.size() + (legacy_rf > 0 ? 1 : 0);  // source codes.size(): the replicas
        const size_t rep_stride = garage_ec_stride_for(stored_max());
        const int quorum = garage_ec_write_quorum(k, m, GARAGE_CONSISTENT);
        uint8_t *blk = dg.conv_blk.get(rep_stride);
        if (!blk) return 0;
        std::atomic<size_t> converted{0};
        for (size_t b0 = 0; b0 < hs.size(); b0 += bmax) {
            const size_t nb = std::min(bmax, hs.size() - b0);
            std::vector<uint8_t> pending(nb, 1);
            for (int c = 1; c < nsrc; c++) {
                const bool rep = c == (int)codes.size();
                const int s_tot = rep ? 1 : codes[c].tot;
                const size_t s_stride = rep ? rep_stride : slot_stride;
                uint8_t *src = dg.conv_src.get(nb * s_tot * s_stride);
                uint8_t *dst = dg.conv_dst.get(nb * tot * (slot_stride + 32));
                if (!src || !dst) break;
                uint8_t *sums = dst + nb * tot * slot_stride;
                std::vector<uint8_t> present(nb * s_tot);
                std::vector<uint32_t> lens(nb);
                // the old stripes (or replicas) of the batch, read by several threads: block j at position j ...
                std::vector<uint8_t> got_src(nb, 0);
                parallel_for(nb, [&](size_t j, std::vector<uint8_t> &) {
                    if (!pending[j]) return;
                    const Hash &h = hs[b0 + j];
                    uint8_t *slot = src + j * s_tot * s_stride;
                    uint32_t len = 0;
                    bool ok = false;
                    uint64_t nbytes = 0;
                    if (rep) {
                        ok = read_replica(h, slot, s_stride, len);
                        nbytes = len;
                    } else {
                        uint8_t *have = present.data() + j * s_tot;
                        gather_into(h, -1, slot, have, len, false, true, nullptr, &ok, &nbytes, c);
                        bool degraded = false;
                        for (int i = 0; i < codes[c].k; i++) degraded |= !have[i];
                        // every survivor whole: the transcode reads what its own plan names (a Clay read set is
                        // whole shards already)
                        if (ok && degraded && !codes[c].clay)
                            gather_into(h, -1, slot, have, len, true, true, nullptr, &ok, &nbytes, c);
                    }
                    convert_bytes_read += nbytes;
                    lens[j] = len;
                    got_src[j] = ok && len > 0 && len <= stored_max();
                });
                // ... then the readable ones packed to the front
                std::vector<size_t> which;  // batch position -> block
                for (size_t j = 0; j < nb; j++) {
                    if (!got_src[j]) continue;
                    const size_t q = which.size();
                    if (q != j) {
                        memmove(src + q * s_tot * s_stride, src + j * s_tot * s_stride, (size_t)s_tot * s_stride);
                        memmove(present.data() + q * s_tot, present.data() + j * s_tot, s_tot);
                        lens[q] = lens[j];
                    }
                    which.push_back(j);
                }
                const size_t n = which.size();
                if (n == 0) continue;
                std::vector<int32_t> status(n, GARAGE_EC_E_UNRECOVERABLE);
                auto t0 = Clock::now();
                int rc = garage_ec_transcode(dg.code_ctx[0], rep ? nullptr : dg.code_ctx[c], src, rep ? nullptr : present.data(),
                                             lens.data(), s_stride, dst, slot_stride, sums, status.data(), n,
                                             GARAGE_EC_MEM_HOST, nullptr);
                convert_call_us += us_since(t0);
                dg.count(n, std::accumulate(lens.begin(), lens.begin() + n, (uint64_t)0));
                if (rc != GARAGE_EC_OK && rc != GARAGE_EC_E_UNRECOVERABLE) continue;
                // the new data shards must hash to the block before anything is written
                std::vector<uint8_t> good(n, 0);
                parallel_for(n, [&](size_t q, std::vector<uint8_t> &tmp) {
                    if (status[q] != GARAGE_EC_OK) return;
                    tmp.resize(lens[q]);
                    assemble(dst + q * tot * slot_stride, lens[q], tmp.data());
                    Hash got;
                    garage_ec_blake2sum(tmp.data(), lens[q], got.data());
                    good[q] = got == hs[b0 + which[q]];
                });
                for (size_t q = 0; q < n; q++) {
                    const Hash &h = hs[b0 + which[q]];
                    if (status[q] != GARAGE_EC_OK) continue;
                    if (!good[q] && !rep) {
                        // a shard of the old stripe passed its tag with other bytes: the hunt quarantines it and
                        // returns the block, which is converted on its own
                        size_t olen = 0;
                        uint32_t l32 = lens[q];
                        int32_t st = 0;
                        if (get_from_stripe(h, blk, stored_max(), &olen, c) == GARAGE_BM_OK && olen == lens[q]) {
                            t0 = Clock::now();
                            rc = garage_ec_transcode(dg.code_ctx[0], nullptr, blk, nullptr, &l32, rep_stride,
                                                     dst + q * tot * slot_stride, slot_stride, sums + q * tot * 32, &st, 1,
                                                     GARAGE_EC_MEM_HOST, nullptr);
                            convert_call_us += us_since(t0);
                            dg.count(1, l32);
                            std::vector<uint8_t> tmp(lens[q]);
                            assemble(dst + q * tot * slot_stride, lens[q], tmp.data());
                            Hash got;
                            garage_ec_blake2sum(tmp.data(), lens[q], got.data());
                            good[q] = rc == GARAGE_EC_OK && got == h;
                        }
                    }
                }
                // the new stripes go to their nodes, several blocks at a time
                parallel_for(n, [&](size_t q, std::vector<uint8_t> &) {
                    if (!good[q]) return;
                    const Hash &h = hs[b0 + which[q]];
                    pending[which[q]] = 0;
                    int who[64];
                    storage_nodes_of(h, who);
                    const size_t L = shard_len_of(lens[q]);
                    int stored = 0;
                    for (int i = 0; i < tot; i++)  // only a durable write counts towards the quorum
                        if (write_shard(who[i], h, i, lens[q], dst + (q * tot + i) * slot_stride, L, sums + (q * tot + i) * 32,
                                        true)) {
                            stored++;
                            convert_bytes_written += L;
                        }
                    {
                        std::lock_guard<std::mutex> lk(refs_mu);
                        refs[h] = lens[q];
                    }
                    if (stored < quorum) {
                        convert_errors++;  // every legacy copy stays; the next sweep tries again
                        return;
                    }
                    convert_blocks++;
                    converted++;
                    for (int i = 0; i < legacy_row(); i++) delete_legacy(ring_node(h, i), h);
                });
            }
            for (size_t j = 0; j < nb; j++) convert_errors += pending[j];
        }
        return converted;
    }
    // fn(i, per-thread scratch) for i < n on up to 16 threads (reads, content hashes and writes of a batch)
    static void parallel_for(size_t n, const std::function<void(size_t, std::vector<uint8_t> &)> &fn)
    {
        const size_t nt = std::min<size_t>(n, std::min(16u, std::max(1u, std::thread::hardware_concurrency())));
        std::atomic<size_t> next{0};
        const RouteTls route = tl_route;  // the workers' GPU work goes to the caller's group
        auto run = [&] {
            tl_route = route;
            std::vector<uint8_t> tmp;
            for (size_t i; (i = next++) < n;) fn(i, tmp);
        };
        std::vector<std::thread> th;
        for (size_t t = 1; t < nt; t++) th.emplace_back(run);
        run();
        for (auto &t : th) t.join();
    }

    // the node that deep-scrubs and stripe-repairs h: the first up node of its row in the newest layout version, -1 if
    // none is up
    int repair_owner(const Hash &h)
    {
        int who[64];
        storage_nodes_of(h, who);
        for (int i = 0; i < tot; i++) {
            Node &nd = *nodes[who[i]];
            std::lock_guard<std::mutex> lk(nd.mu);
            if (nd.up) return who[i];
        }
        return -1;
    }
    // the known blocks not at rc 0 whose repair owner is `node`
    std::vector<Hash> owned_blocks(int node)
    {
        std::vector<Hash> hs;
        {
            std::lock_guard<std::mutex> lk(refs_mu);
            for (auto &kv : refs) {
                auto it = rc.find(kv.first);
                if (it == rc.end() || it->second.count > 0) hs.push_back(kv.first);
            }
        }
        std::vector<Hash> mine;
        for (const Hash &h : hs)
            if (repair_owner(h) == node) mine.push_back(h);
        return mine;
    }

    // garage_bm_deep_scrub_step: see include/garage_block_manager.h and DESIGN.md section 5.4
    int deep_scrub_step(int node, const Hash *cursor, size_t max_blocks, Hash *cursor_out, int *finished,
                        uint64_t *checked, uint64_t *repaired)
    {
        Route route(*this);
        {
            Node &nd = *nodes[node];
            std::lock_guard<std::mutex> lk(nd.mu);
            if (!nd.up) return GARAGE_BM_E_MESSAGE;
        }
        std::vector<Hash> mine = owned_blocks(node);
        sweep_page(mine, cursor, max_blocks, cursor_out, finished);
        uint64_t nchecked = 0, nrep = 0;
        DeviceGroup &dg = grp();
        std::lock_guard<std::mutex> dl(dg.deep_mu);
        const size_t bmax = std::max<uint32_t>(cfg.batch_max_blocks, 1), sbytes = (size_t)tot * slot_stride;
        uint8_t *buf = mine.empty() ? nullptr : dg.deep_buf.get(bmax * (sbytes + 32));
        if (!mine.empty() && !buf) return GARAGE_EC_E_NOMEM;
        const bool multi = multi_version();
        std::vector<uint8_t> blk;
        for (size_t b0 = 0; b0 < mine.size(); b0 += bmax) {
            const size_t nb = std::min(bmax, mine.size() - b0);
            uint8_t *const hashes = buf + bmax * sbytes;
            std::vector<Hash> hv;  // the complete stripes, at buf + i * sbytes
            std::vector<uint32_t> lens;
            std::vector<int> from;  // the node each of their shards came from
            for (size_t b = b0; b < b0 + nb; b++) {
                const Hash &h = mine[b];
                uint8_t *sp = buf + hv.size() * sbytes;
                uint8_t have[GARAGE_EC_MAX_K + GARAGE_EC_MAX_M];
                int src[GARAGE_EC_MAX_K + GARAGE_EC_MAX_M], who[64];
                uint32_t block_len = 0;
                // tags are checked on read; a bad shard is quarantined (and queued) there
                const int got = gather_into(h, -1, sp, have, block_len, /*all=*/true, /*for_gpu=*/true, nullptr, nullptr,
                                            nullptr, 0, src);
                if (got == 0) continue;  // no configured shard: held under a previous code or as replicas
                storage_nodes_of(h, who);
                bool whole = got == tot;
                for (int i = 0; i < tot; i++) {
                    // during a layout change only the newest version's stripe counts: a shard read from an older
                    // holder is missing from it
                    if (have[i] && (!multi || src[i] == who[i])) continue;
                    whole = false;
                    put_to_resync(who[i], h);
                }
                if (!whole) {
                    deep_skipped++;
                    continue;
                }
                memcpy(hashes + hv.size() * 32, h.data(), 32);
                hv.push_back(h);
                lens.push_back(block_len);
                from.insert(from.end(), src, src + tot);
            }
            const size_t nc = hv.size();
            if (!nc) continue;
            std::vector<uint8_t> hash_bad(nc);
            std::vector<uint32_t> mm(nc);
            const auto t0 = Clock::now();
            const int rc_ = garage_ec_deep_check(dg.code_ctx[0], buf, lens.data(), hashes, hash_bad.data(), mm.data(),
                                                 slot_stride, nc, GARAGE_EC_MEM_HOST, nullptr);
            deep_check_us += us_since(t0);
            dg.count(nc, std::accumulate(lens.begin(), lens.end(), (uint64_t)0));
            if (rc_ != GARAGE_EC_OK) return rc_;
            nchecked += nc;
            deep_blocks += nc;
            for (size_t s = 0; s < nc; s++) {
                const Hash &h = hv[s];
                if (!hash_bad[s]) {
                    // the data is right, so every flagged parity is stale: all of them go out before any rebuild (a
                    // Clay repair of one parity reads the others)
                    for (int i = 0; i < m; i++) {
                        if (!((mm[s] >> i) & 1)) continue;
                        quarantine(from[s * tot + k + i], h, 0, multi ? k + i : -1);
                        deep_parity_bad++;
                        nrep++;
                    }
                    continue;
                }
                // the block is wrong: the GET path's hunt finds and quarantines the stale shard, if one set of k is
                // consistent (the stripe's region of the batch buffer is free by now)
                blk.resize(std::max<size_t>(stored_max(), lens[s]));
                size_t out_len = 0;
                if (hunt_stale_shard(h, buf + s * sbytes, blk.data(), blk.size(), &out_len, 0) == GARAGE_BM_OK) nrep++;
                else deep_content_errors++;
            }
        }
        if (checked) *checked = nchecked;
        if (repaired) *repaired = nrep;
        return GARAGE_BM_OK;
    }

    // garage_bm_stripe_repair_step: see include/garage_block_manager.h and DESIGN.md section 5.6
    // garage_bm_set_data_dirs (DESIGN.md section 5.7)
    int set_data_dirs(int node, const garage_bm_data_dir *dirs, int n)
    {
        Node &nd = *nodes[node];
        std::lock_guard<std::mutex> lk(nd.mu);
        if (nd.dir.empty()) return GARAGE_EC_E_INVALID;
        if (!nd.set_drives(dirs, n)) {
            drive_marker_errors++;
            nd.up = false;
            return GARAGE_BM_E_MESSAGE;
        }
        nd.up = true;
        return GARAGE_BM_OK;
    }

    // RebalanceWorker (repair.rs:531-626) over node's drives, in hash order
    int rebalance_step(int node, const Hash *cursor, size_t max_files, Hash *cursor_out, int *finished, uint64_t *moved)
    {
        Node &nd = *nodes[node];
        std::vector<Hash> hs;
        uint64_t gen;
        {
            std::lock_guard<std::mutex> lk(nd.mu);
            if (nd.drives.empty()) return GARAGE_EC_E_INVALID;
            if (!nd.up) return GARAGE_BM_E_MESSAGE;
            nd.misplaced(hs);
            gen = nd.drive_gen;
        }
        int fin = 0;
        sweep_page(hs, cursor, max_files, cursor_out, &fin);
        if (finished) *finished = fin;
        {
            std::lock_guard<std::mutex> lk(rebalance_mu);
            if (!cursor) {
                rebalance_gen[node] = gen + 1;
                rebalance_clean[node] = 1;
            }
        }
        auto allow = [this] { return convert_op_allowed(); };
        uint64_t n = 0;
        bool clean = true;
        std::vector<Hash> bad;
        for (const Hash &h : hs) {
            std::lock_guard<std::mutex> lk(nd.mu);
            if (!nd.up || nd.drive_gen != gen) {
                clean = false;
                break;
            }
            const int prim = nd.drives_of(h)[0];
            for (int d = 0; d < (int)nd.drives.size(); d++) {
                if (d == prim) continue;
                for (const char *ext : {".shard", ".legacy", ""}) {
                    if (!ext[0] && !nd.replicas) continue;
                    uint64_t b = 0;
                    switch (nd.move_to_primary(h, d, ext, allow, &b)) {
                    case Node::kMoved:
                        n++;
                        rebalance_files_moved++;
                        rebalance_bytes_moved += b;
                        break;
                    case Node::kMoveQuarantined:
                        corruption_counter++;
                        bad.push_back(h);
                        break;
                    case Node::kMoveFailed:
                        rebalance_errors++;
                        clean = false;
                        break;
                    default:
                        break;
                    }
                }
            }
        }
        for (const Hash &h : bad) put_to_resync(node, h);
        if (moved) *moved = n;
        std::lock_guard<std::mutex> lk(rebalance_mu);
        if (!clean) rebalance_clean[node] = 0;
        if (!fin) return GARAGE_BM_OK;
        const bool drop = rebalance_gen[node] == gen + 1 && rebalance_clean[node];
        rebalance_gen[node] = 0;
        if (!drop) return GARAGE_BM_OK;
        // every file is in its primary now, and every write since went there: the secondaries can go
        // (without_secondary_locations)
        std::lock_guard<std::mutex> nl(nd.mu);
        if (nd.drive_gen != gen) return GARAGE_BM_OK;
        garage_drive_layout *l = nullptr;
        if (garage_drive_layout_drop_secondaries(&l, nd.dlayout.get()) != GARAGE_LAYOUT_OK) return GARAGE_EC_E_NOMEM;
        std::shared_ptr<garage_drive_layout> keep(l, garage_drive_layout_free);
        std::swap(nd.dlayout, keep);
        if (!nd.save_drives()) {
            std::swap(nd.dlayout, keep);
            return GARAGE_BM_E_MESSAGE;
        }
        nd.drive_gen++;
        return GARAGE_BM_OK;
    }

    int stripe_repair_step(int node, const Hash *cursor, size_t max_blocks, int min_missing, Hash *cursor_out,
                           int *finished, uint64_t *repaired, uint64_t *rebuilt)
    {
        Route route(*this);
        {
            Node &nd = *nodes[node];
            std::lock_guard<std::mutex> lk(nd.mu);
            if (!nd.up) return GARAGE_BM_E_MESSAGE;
        }
        if (multi_version()) return GARAGE_EC_E_INVALID;  // layout sync rebuilds (DESIGN.md section 5.2)
        std::vector<Hash> mine = owned_blocks(node);
        sweep_page(mine, cursor, max_blocks, cursor_out, finished);
        std::vector<RebuildJob> jobs;
        for (const Hash &h : mine) {
            RebuildJob jb;
            jb.h = h;
            jb.grow = true;
            storage_nodes_of(h, jb.to);
            int present = 0, targets = 0;
            for (int i = 0; i < tot; i++) {
                const int p = probe(jb.to[i], h, i);
                present += p > 0;
                if (p == 0) {
                    jb.want[i] = 1;
                    targets++;
                }
            }
            // nothing of the configured code while older copies may exist: the conversion sweep's block
            if (!targets || tot - present < min_missing || (present == 0 && has_legacy())) continue;
            jobs.push_back(jb);
        }
        rebuild_batch(jobs, {stripe_repair_bytes_read, stripe_repair_bytes_fetched, stripe_repair_shards,
                             stripe_repair_bytes_written, stripe_repair_errors, &stripe_repair_call_us, false});
        // stripes their survivors could not rebuild: salvage by segment (DESIGN.md section 5.14)
        for (RebuildJob &jb : jobs) {
            if (jb.written >= 0 || !salvage_possible()) continue;
            SlotLease slot(grp().stripe_slots);
            uint64_t nb = 0;
            const int w = salvage_heal(jb.h, slot.p, -1, &nb);
            if (w > 0) {
                jb.written = w;
                stripe_repair_shards += (uint64_t)w;
                stripe_repair_bytes_written += nb;
            }
        }
        uint64_t nrep = 0, nshards = 0;
        for (const RebuildJob &jb : jobs)
            if (jb.written > 0) {
                nrep++;
                nshards += (uint64_t)jb.written;
            }
        stripe_repairs += nrep;
        if (repaired) *repaired = nrep;
        if (rebuilt) *rebuilt = nshards;
        return GARAGE_BM_OK;
    }

    // garage_bm_convert_step: see include/garage_block_manager.h
    int convert_step(int node, const Hash *cursor, size_t max_blocks, Hash *cursor_out, int *finished, uint64_t *converted)
    {
        Route route(*this);
        Node &nd = *nodes[node];
        std::vector<Hash> hs;
        {
            std::lock_guard<std::mutex> lk(nd.mu);
            if (!nd.up) return GARAGE_BM_E_MESSAGE;
            if (!nd.dir.empty() && has_legacy()) {
                std::vector<Hash> all;
                nd.store_list(all);
                for (const Hash &h : all)
                    if (nd.has_legacy_shard(h) || nd.has_replica(h)) hs.push_back(h);
            }
        }
        sweep_page(hs, cursor, max_blocks, cursor_out, finished);
        std::vector<Hash> todo;
        {
            SlotLease scratch(grp().stripe_slots);  // the quorum check's reads
            for (const Hash &h : hs) {
                {
                    // rc 0: never converted; the legacy copies go once the GC delay has passed, decided and deleted
                    // under both locks like resync_block's offload branch
                    std::lock_guard<std::mutex> rl(refs_mu);
                    auto it = rc.find(h);
                    if (it != rc.end() && it->second.count <= 0) {
                        if (deletable_now(h)) delete_legacy(node, h);
                        continue;
                    }
                }
                if (at_quorum(h, scratch.p, false)) delete_legacy(node, h);  // converted already
                else if (converter_of(h) == node) todo.push_back(h);
            }
        }
        const size_t n = todo.empty() ? 0 : convert_batch(todo);
        if (converted) *converted = n;
        return GARAGE_BM_OK;
    }

    // BlockManager::block_incref / block_decref (manager.rs:452-500), driven in Garage by
    // BlockRefTable::updated (src/model/s3/block_ref_table.rs:69-85): a 0 -> 1 transition queues a
    // resync on every storage node of the block (safety check that the shard really arrives), a
    // drop to 0 queues one too (so that the shard gets deleted once BLOCK_GC_DELAY has passed).
    void block_incref(const Hash &h)
    {
        bool first;
        {
            std::lock_guard<std::mutex> lk(refs_mu);
            RcEntry &c = rc[h];
            first = c.count <= 0;
            c.count = first ? 1 : c.count + 1;
        }
        if (first) queue_on_storage_nodes(h);
    }
    void block_decref(const Hash &h)
    {
        bool zero = false;
        {
            std::lock_guard<std::mutex> lk(refs_mu);
            auto it = rc.find(h);
            if (it == rc.end()) it = rc.emplace(h, RcEntry{1, {}}).first;  // an un-counted block counts as referenced once
            if (it->second.count > 0 && --it->second.count == 0) {
                it->second.zero_since = Clock::now();
                zero = true;
                refs.erase(h);
            }
        }
        if (zero) queue_on_storage_nodes(h);
    }
    void queue_on_storage_nodes(const Hash &h)
    {
        int who[64];
        storage_nodes_of(h, who);
        for (int i = 0; i < tot; i++) put_to_resync(who[i], h);
    }
    int64_t get_block_rc(const Hash &h)
    {
        std::lock_guard<std::mutex> lk(refs_mu);
        auto it = rc.find(h);
        return it == rc.end() ? -1 : it->second.count;
    }

    int resync_all(int node, int workers, uint64_t *resynced)
    {
        Node &nd = *nodes[node];
        std::vector<Hash> todo;
        {
            std::lock_guard<std::mutex> lk(nd.mu);
            for (const auto &q : nd.resync_queue) todo.push_back(q.second);
            nd.resync_queue.clear();
            nd.resync_due.clear();
        }
        std::atomic<size_t> next{0};
        std::atomic<uint64_t> ok{0};
        std::mutex failed_mu;
        std::vector<Hash> failed;
        workers = std::max(1, std::min(workers, 64));
        std::vector<std::thread> th;
        for (int w = 0; w < workers; w++)
            th.emplace_back([&, w] {
                bind_worker(w);
                for (;;) {
                    const size_t i = next++;
                    if (i >= todo.size()) return;
                    int r;
                    try {
                        r = resync_block(node, todo[i]);
                    } catch (...) {
                        r = GARAGE_EC_E_NOMEM;
                    }
                    if (r == GARAGE_BM_OK) {
                        ok++;
                        std::lock_guard<std::mutex> lk(nd.mu);
                        nd.resync_errors.erase(todo[i]);  // an error entry never outlives a success
                    } else {
                        std::lock_guard<std::mutex> lk(failed_mu);
                        failed.push_back(todo[i]);
                    }
                }
            });
        for (auto &t : th) t.join();
        for (const Hash &h : failed) put_to_resync(node, h);  // stays queued (backoff is the caller's)
        if (resynced) *resynced = ok.load();
        return (int)failed.size();
    }

    // ---- scheduled resync (DESIGN.md section 5.8) ---------------------------------------------
    // garage_bm_block_info: see include/garage_block_manager.h
    int block_info(const Hash &h, bool check_tags, garage_bm_block_status *o)
    {
        memset(o, 0, sizeof(*o));
        o->rc = get_block_rc(h);
        o->code = garage_bm_code{k, m, codes[0].l, codes[0].pb ? 1 : 0, codes[0].clay ? 1 : 0};
        o->n_shards = tot;
        uint32_t expect = 0;
        {
            std::lock_guard<std::mutex> lk(refs_mu);
            auto it = refs.find(h);
            if (it != refs.end()) expect = it->second;
        }
        int who[64];
        storage_nodes_of(h, who);
        std::vector<uint8_t> buf(check_tags ? slot_stride : 0);
        uint8_t present[GARAGE_EC_MAX_K + GARAGE_EC_MAX_M] = {0};
        bool all = true;
        for (int i = 0; i < tot; i++) {
            Node &nd = *nodes[who[i]];
            o->node[i] = who[i];
            uint32_t len = 0;
            std::string file;
            Node::ShardPtr sp;
            {
                std::lock_guard<std::mutex> lk(nd.mu);  // headers only: the node's writes wait for no shard read
                o->state[i] = nd.up ? nd.shard_state(h, i, expect, &len, &file, &sp) : GARAGE_BM_SHARD_DOWN;
                auto e = nd.resync_errors.find(h);
                o->resync_errors[i] = e == nd.resync_errors.end() ? 0 : e->second.errors;
            }
            if (check_tags && o->state[i] == GARAGE_BM_SHARD_VALID) o->state[i] = nd.tag_state(i, expect, file, sp, buf);
            present[i] = o->state[i] == GARAGE_BM_SHARD_VALID;
            all = all && present[i];
            if (present[i] && !o->block_len) o->block_len = len;
        }
        // what a rebuild of every shard that is not valid would read: the code's own planner decides recoverability
        uint8_t rd[GARAGE_EC_MAX_K + GARAGE_EC_MAX_M] = {0};
        o->recoverable = all || garage_ec_read_set(codes[0].ctx, present, nullptr, rd) == GARAGE_EC_OK;
        if (!all && o->recoverable) memcpy(o->read_set, rd, tot);
        return GARAGE_BM_OK;
    }

    // <node dir>/resync rewritten from the node's queue and error table (file store, once the node persists them)
    bool save_resync(int node)
    {
        Node &nd = *nodes[node];
        if (nd.dir.empty()) return true;
        std::lock_guard<std::mutex> fl(nd.resync_file_mu);
        std::string img;
        {
            std::lock_guard<std::mutex> lk(nd.mu);
            if (!nd.resync_persist) return true;
            img = nd.resync_image();
        }
        return write_file_atomic(nd.resync_path(), img.data(), img.size(), nullptr, 0, nd.fsync_data, nd.fsync_data);
    }

    // ResyncWorker's iterations (resync.rs:258-336) over the entries of node's queue due now
    int resync_step(int node, int workers, size_t max_blocks, uint64_t *resynced, uint64_t *failed, uint64_t *deferred,
                    int64_t *wait_ms)
    {
        Node &nd = *nodes[node];
        std::lock_guard<std::mutex> sl(nd.resync_step_mu);
        const int64_t now = now_ms();
        std::vector<Hash> todo;
        bool first;
        {
            std::lock_guard<std::mutex> lk(nd.mu);
            if (!nd.up) return GARAGE_BM_E_MESSAGE;
            first = !nd.resync_persist;
            nd.resync_persist = true;
            for (auto it = nd.resync_queue.begin(); it != nd.resync_queue.end() && it->first <= now;) {
                if (max_blocks && todo.size() >= max_blocks) break;
                todo.push_back(it->second);
                nd.resync_due.erase(it->second);
                it = nd.resync_queue.erase(it);
            }
        }
        std::atomic<size_t> next{0};
        std::atomic<uint64_t> n_ok{0}, n_failed{0}, n_deferred{0};
        auto run = [&](int w) {
            bind_worker(w);
            for (size_t i; (i = next++) < todo.size();) {
                const Hash &h = todo[i];
                {
                    std::lock_guard<std::mutex> lk(nd.mu);
                    auto e = nd.resync_errors.find(h);
                    if (e != nd.resync_errors.end() && (uint64_t)now < e->second.next_try()) {  // backing off
                        nd.schedule(h, (int64_t)e->second.next_try());
                        n_deferred++;
                        continue;
                    }
                }
                int64_t gc_wait = 0;
                int r;
                try {
                    r = resync_block(node, h, &gc_wait);
                } catch (...) {
                    r = GARAGE_EC_E_NOMEM;
                }
                std::lock_guard<std::mutex> lk(nd.mu);
                if (r == GARAGE_BM_OK && gc_wait > 0) {  // inside its GC delay: due when it becomes deletable
                    nd.schedule(h, now + gc_wait);
                    n_deferred++;
                } else if (r == GARAGE_BM_OK) {
                    nd.resync_errors.erase(h);
                    n_ok++;
                } else {
                    // Garage stamps last_try = now + 1 so that its re-queue key differs from the entry it removes; this
                    // queue replaces the entry in place, so last_try is the time of the try
                    Node::ResyncError &e = nd.resync_errors[h];
                    e.errors++;
                    e.last_try = (uint64_t)now;
                    e.status = r;
                    nd.schedule(h, (int64_t)e.next_try());
                    n_failed++;
                }
            }
        };
        // every worker is a thread of its own: garage_ec_bind_thread narrows the affinity of the thread it runs on, and
        // the caller's thread keeps its own
        const int nth = (int)std::min<size_t>((size_t)workers, todo.size());
        std::vector<std::thread> th;
        for (int w = 0; w < nth; w++) th.emplace_back(run, w);
        for (auto &t : th) t.join();
        int64_t wait;
        {
            std::lock_guard<std::mutex> lk(nd.mu);
            // IdleFor: until the next entry falls due; 10 s with an empty queue (resync.rs:326-334)
            wait = nd.resync_queue.empty() ? 10000 : std::max<int64_t>(0, nd.resync_queue.begin()->first - now);
        }
        resync_steps++;
        resync_deferred += n_deferred;
        if (resynced) *resynced = n_ok;
        if (failed) *failed = n_failed;
        if (deferred) *deferred = n_deferred;
        if (wait_ms) *wait_ms = wait;
        // a step that took nothing changed nothing the file does not already hold: entries queued since are due now,
        // and the next step that takes them writes
        if (todo.empty() && !first) return GARAGE_BM_OK;
        return save_resync(node) ? GARAGE_BM_OK : GARAGE_BM_E_MESSAGE;
    }

    // list_resync_errors (manager.rs:429-449) of node (-1: every node), in node then hash order
    int list_resync_errors(int node, garage_bm_resync_error *out, size_t cap, size_t *n)
    {
        std::vector<garage_bm_resync_error> all;
        for (int x = node < 0 ? 0 : node; x < (node < 0 ? (int)nodes.size() : node + 1); x++) {
            Node &nd = *nodes[x];
            std::vector<std::pair<Hash, Node::ResyncError>> errs;
            {
                std::lock_guard<std::mutex> lk(nd.mu);
                errs.assign(nd.resync_errors.begin(), nd.resync_errors.end());
            }
            std::sort(errs.begin(), errs.end(), [](const auto &a, const auto &b) { return a.first < b.first; });
            for (const auto &e : errs) {
                garage_bm_resync_error r;
                memset(&r, 0, sizeof(r));
                r.node = x;
                memcpy(r.hash, e.first.data(), 32);
                r.rc = get_block_rc(e.first);
                r.errors = e.second.errors;
                r.last_try_ms = e.second.last_try;
                r.next_try_ms = e.second.next_try();
                r.last_status = e.second.status;
                all.push_back(r);
            }
        }
        *n = all.size();
        if (out && cap) memcpy(out, all.data(), std::min(cap, all.size()) * sizeof(all[0]));
        return GARAGE_BM_OK;
    }

    // clear_backoff (resync.rs:119-134): h (NULL: every errored hash of node) due now, its error count kept
    int resync_retry_now(int node, const Hash *h, uint64_t *n)
    {
        Node &nd = *nodes[node];
        const int64_t now = now_ms();
        uint64_t c = 0;
        {
            std::lock_guard<std::mutex> lk(nd.mu);
            auto clear = [&](const Hash &x, Node::ResyncError &e) {
                e.last_try = (uint64_t)now - e.delay_ms();
                nd.schedule(x, now);
                c++;
            };
            if (h) {
                auto it = nd.resync_errors.find(*h);
                if (it == nd.resync_errors.end() || it->second.errors == 0) return GARAGE_BM_E_MESSAGE;  // not errored
                clear(*h, it->second);
            } else {
                for (auto &e : nd.resync_errors) clear(e.first, e.second);
            }
            nd.resync_persist = true;
        }
        resync_retry_nows += c;
        if (n) *n = c;
        return save_resync(node) ? GARAGE_BM_OK : GARAGE_BM_E_MESSAGE;
    }

    int repair_enqueue_missing(int node, uint64_t *enq)
    {
        std::vector<Hash> all;
        {
            std::lock_guard<std::mutex> lk(refs_mu);
            for (auto &kv : refs) all.push_back(kv.first);
        }
        uint64_t c = 0;
        const bool multi = multi_version();
        for (const Hash &h : all) {
            const int idx = newest_index(h, node);
            if (idx < 0) continue;
            bool has;
            {
                std::lock_guard<std::mutex> lk(nodes[node]->mu);
                has = nodes[node]->store_has(h, multi ? idx : -1);
            }
            if (!has) {
                put_to_resync(node, h);
                c++;
            }
        }
        if (enq) *enq = c;
        return GARAGE_BM_OK;
    }

    // ScrubWorker sweep of one node (repair.rs:438-490) with the GPU computing the shard tags
    // `cursor`/`max_shards`: the scrub iterator checkpoint of the reference (ScrubWorker persists
    // its BlockStoreIterator position every 60 s, repair.rs:186-193,460-464, so a sweep survives a
    // restart): shards are visited in hash order, starting after *cursor (NULL = from the start),
    // at most max_shards of them (0 = all); *cursor_out receives the last hash visited and
    // *finished whether the end of the store was reached.
    int scrub(int node, uint64_t *checked, uint64_t *corrupt, const Hash *cursor = nullptr, size_t max_shards = 0,
              Hash *cursor_out = nullptr, int *finished = nullptr)
    {
        Route route(*this);
        DeviceGroup &dg = grp();
        std::lock_guard<std::mutex> sl(dg.scrub_mu);
        Node &nd = *nodes[node];
        std::vector<Hash> hashes;
        {
            std::lock_guard<std::mutex> lk(nd.mu);
            if (!nd.up) return GARAGE_BM_E_MESSAGE;
            nd.store_list(hashes);
        }
        sweep_page(hashes, cursor, max_shards, cursor_out, finished);
        std::vector<std::pair<Hash, int>> items;  // (hash, Node::ShardFile)
        {
            std::lock_guard<std::mutex> lk(nd.mu);
            for (const Hash &h : hashes)
                for (int f : nd.scrub_files(h)) items.emplace_back(h, f);
        }
        uint64_t nchecked = 0, nbad = 0;
        const size_t chunk = std::max<size_t>(1, (size_t)cfg.batch_max_blocks * tot);
        const size_t stride = slot_stride;
        std::vector<uint8_t> replica;
        for (size_t c0 = 0; c0 < items.size(); c0 += chunk) {
            const size_t n = std::min(chunk, items.size() - c0);
            uint8_t *buf = dg.scrub_buf.get(n * stride + n * 32 + n + n * 4);
            if (!buf) return GARAGE_EC_E_NOMEM;
            uint8_t *expect = buf + n * stride, *bad = expect + n * 32;
            std::vector<uint32_t> lens(n, 0);
            std::vector<uint8_t> state(n, 0);  // 0 gone, 1 to be checked on the GPU, 2 corrupt already, 3 checked on the CPU
            {
                std::lock_guard<std::mutex> lk(nd.mu);
                for (size_t i = 0; i < n; i++) {
                    ShardMeta mt;
                    memset(expect + i * 32, 0, 32);
                    const Hash &h = items[c0 + i].first;
                    const int kind = items[c0 + i].second;
                    ReadResult r;
                    if (kind == Node::kReplicaFile) {  // a replica is checked against its content hash
                        replica.resize(stored_max());
                        uint32_t len = 0;
                        r = nd.replica_read_into(h, replica.data(), replica.size(), len);
                        if (r == kReadMissing) continue;
                        Hash got;
                        if (r == kReadOk) {
                            bytes_read += len;
                            garage_ec_blake2sum(replica.data(), len, got.data());
                        }
                        state[i] = r == kReadOk && got == h ? 3 : 2;
                        continue;
                    }
                    r = nd.scrub_read_into(h, kind, buf + i * stride, stride, mt);
                    if (r == kReadMissing) continue;
                    if (r == kReadInvalid) {
                        state[i] = 2;
                        continue;
                    }
                    lens[i] = mt.shard_len;
                    bytes_read += mt.shard_len;
                    if (mt.sum_kind == sum_kind) {
                        memcpy(expect + i * 32, mt.sum.data(), 32);
                        state[i] = 1;
                    } else {  // written under another tag kind: check it on the CPU
                        Hash got;
                        garage_ec_shard_sum_host(mt.sum_kind, buf + i * stride, mt.shard_len, got.data());
                        state[i] = got == mt.sum ? 3 : 2;
                        lens[i] = 0;
                    }
                }
            }
            int rc = garage_ec_check_sums(dg.code_ctx[0], buf, expect, lens.data(), stride, n, 1, bad, GARAGE_EC_MEM_HOST,
                                          nullptr);
            if (rc != GARAGE_EC_OK) return rc;
            dg.count(n, std::accumulate(lens.begin(), lens.end(), (uint64_t)0));
            for (size_t i = 0; i < n; i++) {
                if (!state[i]) continue;
                nchecked++;
                if (state[i] == 3 || (state[i] == 1 && !bad[i])) continue;
                nbad++;
                quarantine(node, items[c0 + i].first, 0, -1, items[c0 + i].second,
                           state[i] == 1 && items[c0 + i].second == Node::kShardFile);  // tag failed on the GPU
            }
        }
        scrub_checked += nchecked;
        scrub_corrupt += nbad;
        if (checked) *checked = nchecked;
        if (corrupt) *corrupt = nbad;
        return GARAGE_BM_OK;
    }

    // worker thread w of a resync pass or a load run: on the CPUs of the node of group w mod n, so that the workers of
    // a pass spread over the listed devices' sockets and each is routed to a group of its own socket
    void bind_worker(int w) const { garage_ec_bind_thread(groups[(size_t)w % groups.size()]->code_ctx[0]); }

    // ---- native closed-loop load generator (tools/bm_bench.py drives it): `threads` client threads,
    // each PUTs (mode 0) or GETs (mode 1) `per_thread` blocks of `block_len` bytes.  Blocks are the
    // splitmix64 stream (seed, thread, i); hashing them is the S3 layer's job (put.rs:448) and
    // happens before the clock starts.
    int bench(int threads, int per_thread, uint32_t block_len, int mode, uint64_t seed, double *gib_per_s, uint64_t *errors)
    {
        if (threads < 1 || per_thread < 1 || block_len < 1 || shard_len_of(block_len) > slot_stride) return GARAGE_EC_E_INVALID;
        const size_t nb = (size_t)threads * per_thread;
        std::vector<uint8_t> data;
        std::vector<Hash> hashes(nb);
        const size_t words = ((size_t)block_len + 7) / 8;
        if (mode == 0) data.resize(nb * words * 8);
        auto gen = [&](size_t b, uint8_t *dst) {
            uint64_t *w = reinterpret_cast<uint64_t *>(dst);
            for (size_t i = 0; i < words; i++) {
                uint64_t z = seed + (b * words + i + 1) * 0x9E3779B97F4A7C15ull;
                z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
                z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
                w[i] = z ^ (z >> 31);
            }
        };
        {
            std::vector<std::thread> th;
            for (int t = 0; t < threads; t++)
                th.emplace_back([&, t] {
                    std::vector<uint8_t> tmp(words * 8);
                    for (int i = 0; i < per_thread; i++) {
                        const size_t b = (size_t)t * per_thread + i;
                        uint8_t *dst = mode == 0 ? data.data() + b * words * 8 : tmp.data();
                        gen(b, dst);
                        garage_ec_blake2sum(dst, block_len, hashes[b].data());
                    }
                });
            for (auto &x : th) x.join();
        }
        if (mode == 0 && !warmed.exchange(true)) {
            // first use of this manager: one block through every dispatcher (streams, lane buffers, kernels)
            std::vector<uint8_t> wblk(words * 8);
            gen(nb, wblk.data());
            Hash wh;
            garage_ec_blake2sum(wblk.data(), block_len, wh.data());
            std::vector<std::thread> wt;
            for (int t = 0; t < 3 * DeviceGroup::kWorkers * (int)groups.size(); t++)
                wt.emplace_back([&, t] {
                    bind_worker(t);
                    try {
                        rpc_put_block(wh, wblk.data(), block_len);
                    } catch (...) {
                    }
                });
            for (auto &x : wt) x.join();
        }
        if (mode == 0 && nodes[0]->dir.empty())  // the stores' memory is in place before the clock starts (see ShardArena)
            ShardArena::instance().reserve(shard_len_of(block_len), nb * (size_t)tot);
        std::atomic<uint64_t> errs{0};
        std::atomic<int> ready{0};
        std::atomic<bool> go{false};
        std::vector<std::thread> th;
        for (int t = 0; t < threads; t++)
            th.emplace_back([&, t] {
                bind_worker(t);
                std::vector<uint8_t> out(mode == 1 ? block_len : 0);
                ready++;
                while (!go.load(std::memory_order_acquire)) std::this_thread::yield();
                for (int i = 0; i < per_thread; i++) {
                    const size_t b = (size_t)t * per_thread + i;
                    int rc;
                    try {
                        if (mode == 0) {
                            rc = rpc_put_block(hashes[b], data.data() + b * words * 8, block_len);
                        } else {
                            size_t n = 0;
                            rc = rpc_get_block(hashes[b], out.data(), out.size(), &n);
                            if (rc == GARAGE_BM_OK && n != block_len) rc = GARAGE_BM_E_CORRUPT_DATA;
                        }
                    } catch (...) {
                        rc = GARAGE_EC_E_NOMEM;
                    }
                    if (rc != GARAGE_BM_OK) errs++;
                }
            });
        while (ready.load() < threads) std::this_thread::yield();
        const auto t0 = Clock::now();
        go.store(true, std::memory_order_release);
        for (auto &x : th) x.join();
        const double el = std::chrono::duration<double>(Clock::now() - t0).count();
        if (gib_per_s) *gib_per_s = (double)nb * block_len / el / (double)(1ull << 30);
        if (errors) *errors = errs.load();
        return GARAGE_BM_OK;
    }
};

// ================================================================= C API
// Nothing throws across the C boundary (the reference returns Result everywhere,
// src/util/error.rs:14-82): allocation failures and anything unexpected become status codes.
#define BM_GUARD(expr)                       \
    try {                                    \
        return (expr);                       \
    } catch (const std::bad_alloc &) {       \
        return GARAGE_EC_E_NOMEM;            \
    } catch (...) {                          \
        return GARAGE_BM_E_MESSAGE;          \
    }

// the resumable sweeps: the cursor in and out of one garage_bm_*_step call
template <class Step>
static int bm_step(garage_bm *bm, int node, const uint8_t *cursor32, uint8_t *cursor_out32, Step step)
{
    if (!bm || node < 0 || node >= (int)bm->nodes.size()) return GARAGE_EC_E_INVALID;
    BM_GUARD(([&] {
        Hash cur, out;
        if (cursor32) cur = to_hash(cursor32);
        const int rc = step(cursor32 ? &cur : nullptr, &out);
        if (rc == GARAGE_BM_OK && cursor_out32) memcpy(cursor_out32, out.data(), 32);
        return rc;
    }()));
}

extern "C" {

void garage_bm_default_config(garage_bm_config *c)
{
    if (!c) return;
    c->data_shards = 10;
    c->parity_shards = 4;
    c->cuda_device = 0;
    c->n_nodes = 14;
    c->block_size = 1u << 20;               // util/config.rs:273-275
    c->block_ram_buffer_max = 256ull << 20;  // util/config.rs:276-278
    c->batch_max_blocks = 64;
    c->batch_linger_us = 100;  // a longer linger costs closed-loop PUT rate at 32 callers
    c->data_dir = nullptr;
    c->shard_sum_kind = GARAGE_EC_SUM_ADLER8;
    c->verify_content_hash = 1;
    c->data_fsync = 0;             // util/config.rs data_fsync default
    c->block_gc_delay_ms = 600000;  // BLOCK_GC_DELAY, manager.rs:49-52
    c->local_groups = 0;            // RS
    c->piggyback = 0;
    c->previous_codes = nullptr;    // no code change in progress
    c->n_previous_codes = 0;
    c->legacy_replicas = 0;
    c->layout = nullptr;            // the fixed ring
    c->clay = 0;                    // not Clay
    c->clay_layout = 0;             // a Clay store keeps the fixed ring
}

// a code garage_ec_create / _lrc / _piggyback / _clay accepts, with tags the block manager can check; the rules of the
// configured code and of every previous code (PB: 1 <= k <= 16, 2 <= m <= 4, no LRC groups, and adler8 tags for its
// half reads; Clay: k >= 2, 2 <= m <= 4, alpha = m^ceil((k+m)/m) <= 256, neither LRC groups nor PB)
static bool code_ok(int k, int m, int l, int piggyback, int clay, int sum_kind)
{
    if (k < 1 || m < 1 || k > GARAGE_EC_MAX_K || m > GARAGE_EC_MAX_M) return false;
    if (l < 0 || (l > 0 && (l >= m || k % l))) return false;
    if ((piggyback != 0 && piggyback != 1) || (clay != 0 && clay != 1)) return false;
    if (clay) {
        int alpha = 1;
        for (int t = (k + m + m - 1) / m; t > 0 && alpha <= 256; t--) alpha *= m;
        return m >= 2 && m <= 4 && k >= 2 && alpha <= 256 && !piggyback && l == 0;
    }
    return !piggyback || (l == 0 && k <= 16 && m >= 2 && m <= 4 && sum_kind != GARAGE_EC_SUM_BLAKE2);
}

// a data_dir list garage_bm_create and garage_bm_set_data_dirs take: 1..GARAGE_BM_MAX_DATA_DIRS entries with relative
// paths inside the node directory, distinct once normalised, capacity > 0 unless read-only, and at least one with
// capacity (the drive layout's own rules)
static bool drive_list_ok(const garage_bm_data_dir *d, int n)
{
    if (n < 1 || n > GARAGE_BM_MAX_DATA_DIRS || !d) return false;
    std::vector<std::string> seen;
    std::vector<uint64_t> cap(n);
    for (int i = 0; i < n; i++) {
        if (!d[i].path || !d[i].path[0] || d[i].path[0] == '/' || (d[i].read_only != 0 && d[i].read_only != 1)) return false;
        if (!d[i].read_only && d[i].capacity == 0) return false;
        const std::string p = Node::normal_path(d[i].path);
        if (p == ".." || p.compare(0, 3, "../") == 0 || std::find(seen.begin(), seen.end(), p) != seen.end()) return false;
        seen.push_back(p);
        cap[i] = d[i].read_only ? 0 : d[i].capacity;
    }
    garage_drive_layout *l = nullptr;
    const int rc = garage_drive_layout_init(&l, n, cap.data(), nullptr);
    garage_drive_layout_free(l);
    return rc == GARAGE_LAYOUT_OK;
}

// a context running code `c` (RS, LRC, PB or Clay) with shard tags of `sum_kind`
static int create_ctx(const CodeDesc &c, int device, int sum_kind, garage_ec_ctx **out)
{
    const int rc = c.clay ? garage_ec_create_clay(out, device, c.k, c.m, GARAGE_EC_VANDERMONDE)
                   : c.pb ? garage_ec_create_piggyback(out, device, c.k, c.m, GARAGE_EC_VANDERMONDE)
                   : c.l  ? garage_ec_create_lrc(out, device, c.k, c.l, c.m - c.l)
                          : garage_ec_create(out, device, c.k, c.m, GARAGE_EC_VANDERMONDE);
    if (rc == GARAGE_EC_OK) garage_ec_set_sum_kind(*out, sum_kind);
    return rc;
}

// The group of bm on `device` (DESIGN.md section 5.13): a context per code (the first group takes the codes' own), the
// dispatcher contexts and their parity buffers, the pools on the device's NUMA node, every context warmed, then the
// dispatcher threads.  What it built before a failure is torn down with the manager.
static int create_group(garage_bm *bm, int device, bool first)
{
    bm->groups.emplace_back(new DeviceGroup());
    DeviceGroup &g = *bm->groups.back();
    g.device = device;
    const garage_bm_config &cfg = bm->cfg;
    const int m = bm->m;
    int rc = GARAGE_EC_OK;
    for (const auto &c : bm->codes) {
        garage_ec_ctx *x = first ? c.ctx : nullptr;
        if (!first && (rc = create_ctx(c, device, bm->sum_kind, &x)) != GARAGE_EC_OK) return rc;
        g.code_ctx.push_back(x);
    }
    garage_ec_ctx *const ec = g.code_ctx[0];
    garage_ec_numa_info(ec, &g.numa_node, nullptr);
    for (PinnedBuf *b : {&g.scrub_buf, &g.deep_buf, &g.conv_src, &g.conv_dst, &g.conv_blk}) b->ctx = ec;
    for (int w = 0; w < DeviceGroup::kWorkers; w++) {
        rc = create_ctx(bm->codes[0], device, bm->sum_kind, &g.enc_ctx[w]);
        if (rc == GARAGE_EC_OK) rc = create_ctx(bm->codes[0], device, bm->sum_kind, &g.rec_ctx[w]);
        if (rc != GARAGE_EC_OK) return rc;
        // Dispatchers wait for their batch spinning in the driver (default) or sleeping on an event
        // (GARAGE_BM_SLEEP_WAIT=1).  With 32 client threads on a 16-CPU host PUT is faster spinning: the wake-up
        // latency costs more than the three CPUs.
        const int sleep_wait = getenv("GARAGE_BM_SLEEP_WAIT") ? 1 : 0;
        garage_ec_set_wait_mode(g.enc_ctx[w], sleep_wait);
        garage_ec_set_wait_mode(g.rec_ctx[w], sleep_wait);
        for (auto &eb : g.enc_out[w]) eb.ctx = g.enc_ctx[w];
        // the pinned parity buffers at their final size now, not on the first large batch
        const size_t out_bytes = (size_t)std::max<uint32_t>(cfg.batch_max_blocks, 1) * ((size_t)m * bm->slot_stride + (size_t)bm->tot * 32);
        for (auto &eb : g.enc_out[w])
            if (!eb.get(out_bytes)) return GARAGE_EC_E_NOMEM;
    }
    const size_t nslots = (size_t)std::max<uint32_t>(cfg.batch_max_blocks, 1) * (DeviceGroup::kWorkers + 1);
    if (!g.put_slots.init(ec, nslots, cfg.block_size)) return GARAGE_EC_E_NOMEM;
    int max_tot = bm->tot;  // a stripe slot holds a stripe of any code in play
    for (const auto &c : bm->codes) max_tot = std::max(max_tot, c.tot);
    if (!g.stripe_slots.init(ec, nslots, (size_t)max_tot * bm->slot_stride)) return GARAGE_EC_E_NOMEM;
    garage_ec_numa_info(ec, nullptr, &g.pool_node);
    // Warm every dispatcher's context now: streams, lane buffers, and the first launch of each kernel (CUDA
    // loads kernels lazily) cost tens of milliseconds that would otherwise land on the first real batches.
    {
        SlotLease blk(g.put_slots), stripe(g.stripe_slots);
        const uint32_t wlen = cfg.block_size;
        memset(blk.p, 0x5a, wlen);
        memset(stripe.p, 0, (size_t)bm->tot * bm->slot_stride);
        for (int w = 0; w < DeviceGroup::kWorkers; w++) {
            const uint8_t *ptrs[1] = {blk.p};
            uint8_t *par = g.enc_out[w][0].get(1);
            rc = garage_ec_encode_blocks_with_sums(g.enc_ctx[w], ptrs, &wlen, 1, par, par + (size_t)m * bm->slot_stride, bm->slot_stride);
            if (rc != GARAGE_EC_OK) return rc;
            uint8_t present[GARAGE_EC_MAX_K + GARAGE_EC_MAX_M], want[GARAGE_EC_MAX_K + GARAGE_EC_MAX_M] = {0};
            memset(present, 1, sizeof(present));
            present[0] = 0;
            want[0] = 1;
            uint8_t *stripes[1] = {stripe.p};
            const uint32_t slen = (uint32_t)bm->shard_len_of(wlen);
            int32_t st = 0;
            rc = garage_ec_reconstruct_stripes(g.rec_ctx[w], stripes, present, want, &st, &slen, bm->slot_stride, 1);
            if (rc != GARAGE_EC_OK) return rc;
        }
        uint8_t bad1 = 0, exp1[32] = {0};
        const uint32_t slen = (uint32_t)bm->shard_len_of(wlen);
        rc = garage_ec_check_sums(ec, stripe.p, exp1, &slen, bm->slot_stride, 1, 1, &bad1, GARAGE_EC_MEM_HOST, nullptr);
        if (rc != GARAGE_EC_OK) return rc;
    }
    // the dispatchers run on the device's node and route their own work to their group
    DeviceGroup *gp = &g;
    auto start = [bm, gp] {
        garage_ec_bind_thread(gp->code_ctx[0]);
        tl_route = {bm, gp};
    };
    g.enc_batcher.reset(new Batcher<EncodeItem>(cfg.batch_max_blocks, cfg.batch_linger_us, DeviceGroup::kWorkers,
                                                [bm](int w, std::vector<EncodeItem *> &b) { bm->run_encode(w, b); }, start));
    g.rec_batcher.reset(new Batcher<ReconItem>(cfg.batch_max_blocks, cfg.batch_linger_us, DeviceGroup::kWorkers,
                                               [bm](int w, std::vector<ReconItem *> &b) { bm->run_reconstruct(w, b); }, start));
    return GARAGE_EC_OK;
}

// devices: the listed devices, one group each.  check_range: a device past garage_ec_device_count is refused before any
// CUDA context exists (garage_bm_create leaves that to the context's own NODEVICE, as it always has).
static int bm_create(garage_bm **out, const garage_bm_config *cfg, const garage_bm_data_dir *data_dirs, int n_data_dirs,
                     const int *devices, int n_devices, bool check_range)
{
    *out = nullptr;
    const int k = cfg->data_shards, m = cfg->parity_shards, l = cfg->local_groups;
    if (!code_ok(k, m, l, cfg->piggyback, cfg->clay, cfg->shard_sum_kind) || cfg->n_nodes < k + m || cfg->n_nodes > 256)
        return GARAGE_EC_E_INVALID;
    if (cfg->shard_sum_kind != GARAGE_EC_SUM_BLAKE2 && cfg->shard_sum_kind != GARAGE_EC_SUM_ADLER8) return GARAGE_EC_E_INVALID;
    const bool pb = cfg->piggyback != 0;
    // a Clay store changes its layout only with clay_layout
    const bool clay = cfg->clay != 0;
    if ((cfg->clay_layout != 0 && cfg->clay_layout != 1) || (cfg->clay_layout && !clay)) return GARAGE_EC_E_INVALID;
    if (clay && cfg->layout && !cfg->clay_layout) return GARAGE_EC_E_INVALID;
    // previous codes and replicas (all checked before any CUDA call)
    const int np = cfg->n_previous_codes;
    if (np < 0 || np > GARAGE_BM_MAX_PREVIOUS_CODES || (np > 0 && !cfg->previous_codes)) return GARAGE_EC_E_INVALID;
    if (cfg->legacy_replicas < 0 || cfg->legacy_replicas > cfg->n_nodes) return GARAGE_EC_E_INVALID;
    for (int i = 0; i < np; i++) {
        const garage_bm_code &p = cfg->previous_codes[i];
        if (!code_ok(p.k, p.m, p.local_groups, p.piggyback, p.clay, cfg->shard_sum_kind) || p.k + p.m > cfg->n_nodes)
            return GARAGE_EC_E_INVALID;
        if (p.k == k && p.m == m && p.local_groups == l && (p.piggyback != 0) == pb && (p.clay != 0) == clay)
            return GARAGE_EC_E_INVALID;
        for (int j = 0; j < i; j++) {
            const garage_bm_code &q = cfg->previous_codes[j];
            if (p.k == q.k && p.m == q.m && p.local_groups == q.local_groups && p.piggyback == q.piggyback && p.clay == q.clay)
                return GARAGE_EC_E_INVALID;
        }
    }
    // drives: a file store only, and a list the drive layout takes
    if (n_data_dirs < 0 || (n_data_dirs > 0 && (!(cfg->data_dir && cfg->data_dir[0]) || !drive_list_ok(data_dirs, n_data_dirs))))
        return GARAGE_EC_E_INVALID;
    // the layout history: <data_dir>/layout wins over cfg->layout; both are checked before any CUDA call
    auto lays = std::make_shared<garage_bm::Layouts>();
    std::vector<uint64_t> synced(cfg->n_nodes, 0);
    const bool file_store = cfg->data_dir && cfg->data_dir[0];
    const std::string layout_path = file_store ? std::string(cfg->data_dir) + "/layout" : std::string();
    if (cfg->layout && !garage_bm::layout_from_spec(*lays, 1, cfg->n_nodes, k, m, cfg->layout, nullptr)) return GARAGE_EC_E_INVALID;
    bool layout_file = file_store && cfg->layout;
    if (file_store) {
        auto loaded = std::make_shared<garage_bm::Layouts>();
        const int r = garage_bm::load_layout(layout_path, cfg->n_nodes, k + m, *loaded, synced);
        if (r < 0) return GARAGE_EC_E_INVALID;
        if (r > 0) {
            lays = loaded;
            layout_file = true;
        }
    }
    // a store changes its layout or its code, not both at once
    if (lays->v.size() > 1 && (np > 0 || cfg->legacy_replicas > 0)) return GARAGE_EC_E_INVALID;
    if (clay && layout_file && !cfg->clay_layout) return GARAGE_EC_E_INVALID;  // a Clay store keeps the fixed ring
    // with no device at all, the first context's NODEVICE is the answer, as for garage_bm_create
    const int ndev = check_range ? garage_ec_device_count() : 0;
    for (int i = 0; i < n_devices; i++)
        if (ndev > 0 && devices[i] >= ndev) return GARAGE_EC_E_INVALID;
    std::unique_ptr<garage_bm> bm(new garage_bm());
    bm->cfg = *cfg;
    if (!bm->cfg.block_size) bm->cfg.block_size = 1u << 20;
    bm->k = k;
    bm->m = m;
    bm->tot = k + m;
    bm->sum_kind = cfg->shard_sum_kind;
    bm->legacy_rf = cfg->legacy_replicas;
    bm->cfg.previous_codes = nullptr;  // not kept: the caller's array may go away
    // codes[0] the configured code (every dispatcher context runs it too), then one context per previous code, same
    // tag kind and matrices as the configured one
    bm->codes.resize(1 + np);
    int rc = GARAGE_EC_OK;
    for (int i = 0; i <= np; i++) {
        garage_bm::Code &c = bm->codes[i];
        const garage_bm_code p = i ? cfg->previous_codes[i - 1] : garage_bm_code{k, m, l, cfg->piggyback, cfg->clay};
        c.k = p.k;
        c.m = p.m;
        c.l = p.local_groups;
        c.pb = p.piggyback != 0;
        c.clay = p.clay != 0;
        c.tot = p.k + p.m;
        rc = create_ctx(c, devices[0], bm->sum_kind, &c.ctx);
        if (rc != GARAGE_EC_OK) {  // no GPU => no block manager: there is no CPU fallback
            garage_bm_destroy(bm.release());
            return rc;
        }
        c.quantum = c.pb ? 128u : 1u;
        if (c.clay) {
            int alpha = 0;
            garage_ec_clay_info(c.ctx, nullptr, nullptr, &alpha, nullptr, nullptr);
            c.quantum = 16u * (uint32_t)alpha;
        }
        // slots and the scrub buffer hold a shard of the largest code in play
        bm->slot_stride = std::max(bm->slot_stride, garage_ec_stride_for((uint32_t)bm->shard_len_of(bm->stored_max(), i)));
    }
    if (lays->v.empty() && cfg->n_nodes <= GARAGE_LAYOUT_MAX_NODES) {
        const int n = cfg->n_nodes, tot = k + m;
        std::vector<uint8_t> ring((size_t)GARAGE_NB_PARTITIONS * tot);
        for (int p = 0; p < GARAGE_NB_PARTITIONS; p++)
            for (int i = 0; i < tot; i++) ring[(size_t)p * tot + i] = (uint8_t)((p % n + i) % n);
        std::vector<int32_t> zone(n, 0);
        std::vector<uint64_t> capacity(n, 1);
        garage_layout *l = nullptr;
        if (garage_layout_from_ring(&l, 1, n, zone.data(), capacity.data(), tot, ring.data()) == GARAGE_LAYOUT_OK) {
            lays->v.emplace_back(l, garage_layout_free);
            lays->zone.push_back(std::move(zone));
            lays->capacity.push_back(std::move(capacity));
        }
    }
    bm->layouts_ = lays;
    bm->layout_file = layout_file;
    bm->layout_path = layout_path;
    bm->synced = synced;
    bm->pass_version.assign(cfg->n_nodes, 0);
    bm->pass_clean.assign(cfg->n_nodes, 0);
    bm->cfg.layout = nullptr;  // not kept: the caller's spec may go away
    bm->rebalance_gen.assign(cfg->n_nodes, 0);
    bm->rebalance_clean.assign(cfg->n_nodes, 0);
    for (int i = 0; i < cfg->n_nodes; i++) {
        bm->nodes.emplace_back(new Node());
        Node &nd = *bm->nodes.back();
        nd.codes.assign(1, bm->codes[0]);
        nd.fsync_data = cfg->data_fsync != 0;
        if (cfg->data_dir && cfg->data_dir[0]) {
            nd.dir = std::string(cfg->data_dir) + "/node" + std::to_string(i);
            nd.by_index = layout_file;
            nd.codes.assign(bm->codes.begin(), bm->codes.end());  // previous codes exist on disk only
            nd.replicas = bm->legacy_rf > 0;
            std::error_code ec;
            std::filesystem::create_directories(nd.dir, ec);
            // drives: <node dir>/data_layout wins over the configured list, which seeds a node without one
            const int lr = nd.load_drives();
            if (lr < 0) {
                garage_bm_destroy(bm.release());
                return GARAGE_EC_E_INVALID;
            }
            bool markers_ok = true;
            if (lr == 0 && n_data_dirs > 0) {
                markers_ok = nd.set_drives(data_dirs, n_data_dirs);
            } else if (lr > 0) {
                std::vector<Node::Drive> ds = nd.drives;
                markers_ok = Node::check_markers(ds);
                bool recorded = false;
                for (size_t d = 0; markers_ok && d < ds.size(); d++) recorded = recorded || ds[d].marker != nd.drives[d].marker;
                if (recorded) {
                    nd.drives = ds;
                    markers_ok = nd.save_drives();
                }
            }
            if (!markers_ok) {  // Garage refuses to start on an unmounted or swapped disk
                nd.up = false;
                bm->drive_marker_errors++;
            }
            // restart: what is on disk is what exists (the block_ref table would say the same), shards of previous
            // codes and replicas included
            nd.resync_persist = nd.load_resync();  // the scheduled queue and error table of an earlier run
            std::vector<Hash> have;
            nd.store_list(have);
            std::vector<uint8_t> tmp(bm->slot_stride);
            for (const Hash &h : have) {
                uint32_t len = 0;
                if (nd.block_len_of(h, tmp, bm->stored_max(), bm->refs.count(h) != 0, len)) bm->refs[h] = len;
            }
        }
    }
    bm->ram.reset(new ByteSemaphore(cfg->block_ram_buffer_max ? cfg->block_ram_buffer_max : (256ull << 20)));
    auto destroy_on_error = [&](int code) {
        garage_bm_destroy(bm.release());
        return code;
    };
    // a layout given in the configuration is recorded, so that a restart keeps it and its later versions
    if (layout_file && !std::filesystem::exists(layout_path) && !bm->save_layout(*lays)) return destroy_on_error(GARAGE_BM_E_MESSAGE);
    for (int i = 0; i < n_devices; i++) {
        rc = create_group(bm.get(), devices[i], i == 0);
        if (rc != GARAGE_EC_OK) return destroy_on_error(rc);  // no group left out: all of them or no manager
    }
    *out = bm.release();
    return GARAGE_BM_OK;
}

int garage_bm_create(garage_bm **out, const garage_bm_config *cfg)
{
    if (!out || !cfg) return GARAGE_EC_E_INVALID;
    BM_GUARD(bm_create(out, cfg, nullptr, 0, &cfg->cuda_device, 1, false));
}

int garage_bm_create_with_drives(garage_bm **out, const garage_bm_config *cfg, const garage_bm_data_dir *data_dirs,
                                 int n_data_dirs)
{
    if (!out || !cfg) return GARAGE_EC_E_INVALID;
    BM_GUARD(bm_create(out, cfg, data_dirs, n_data_dirs, &cfg->cuda_device, 1, false));
}

int garage_bm_create_on_devices(garage_bm **out, const garage_bm_config *cfg, const garage_bm_data_dir *data_dirs,
                                int n_data_dirs, const int *cuda_devices, int n_devices)
{
    if (!out || !cfg) return GARAGE_EC_E_INVALID;
    *out = nullptr;
    if (!cuda_devices || n_devices < 1 || n_devices > GARAGE_BM_MAX_DEVICES) return GARAGE_EC_E_INVALID;
    for (int i = 0; i < n_devices; i++)
        if (cuda_devices[i] < 0) return GARAGE_EC_E_INVALID;
    BM_GUARD(bm_create(out, cfg, data_dirs, n_data_dirs, cuda_devices, n_devices, true));
}

void garage_bm_destroy(garage_bm *bm)
{
    if (!bm) return;
    for (int i = 0; i < (int)bm->nodes.size(); i++) {  // the scheduled queues of the nodes that keep them
        try {
            bm->save_resync(i);
        } catch (...) {
        }
    }
    for (auto &g : bm->groups) {  // every dispatcher joined before any pinned memory goes
        g->enc_batcher.reset();
        g->rec_batcher.reset();
    }
    std::vector<garage_ec_ctx *> ctxs;  // each once: the first group's code contexts are the codes' own
    for (auto &g : bm->groups) {
        g->stop();  // pinned memory goes before its context
        ctxs.insert(ctxs.end(), std::begin(g->enc_ctx), std::end(g->enc_ctx));
        ctxs.insert(ctxs.end(), std::begin(g->rec_ctx), std::end(g->rec_ctx));
        ctxs.insert(ctxs.end(), g->code_ctx.begin(), g->code_ctx.end());
    }
    for (const auto &c : bm->codes) ctxs.push_back(c.ctx);
    delete bm;
    std::sort(ctxs.begin(), ctxs.end());
    ctxs.erase(std::unique(ctxs.begin(), ctxs.end()), ctxs.end());
    for (garage_ec_ctx *c : ctxs)
        if (c) garage_ec_destroy(c);
}

int garage_bm_get_device_metrics(garage_bm *bm, garage_bm_device_metrics *out, int cap, int *n)
{
    if (!bm || !n || cap < 0 || (!out && cap > 0)) return GARAGE_EC_E_INVALID;
    *n = (int)bm->groups.size();
    for (int i = 0; i < *n && i < cap; i++) {
        const DeviceGroup &g = *bm->groups[i];
        garage_bm_device_metrics &o = out[i];
        o.cuda_device = g.device;
        o.numa_node = g.numa_node;
        o.batches = g.batches;
        o.blocks = g.blocks;
        o.bytes = g.bytes;
        o.routed_local = g.routed_local;
        o.routed_remote = g.routed_remote;
        o.pool_numa_node = g.pool_node;
    }
    return GARAGE_BM_OK;
}

void garage_bm_blake2sum(const uint8_t *data, size_t len, uint8_t hash_out[32]) { garage_ec_blake2sum(data, len, hash_out); }

int garage_bm_rpc_put_block(garage_bm *bm, const uint8_t hash[32], const uint8_t *data, size_t len)
{
    if (!bm || !hash || !data) return GARAGE_EC_E_INVALID;
    BM_GUARD(bm->rpc_put_block(to_hash(hash), data, len));
}

int garage_bm_rpc_get_block(garage_bm *bm, const uint8_t hash[32], uint8_t *out, size_t cap, size_t *out_len)
{
    if (!bm || !hash || !out_len || !out) return GARAGE_EC_E_INVALID;
    BM_GUARD(bm->rpc_get_block(to_hash(hash), out, cap, out_len));
}

int garage_bm_rpc_put_block_sealed(garage_bm *bm, const uint8_t *key32, const uint8_t *data, size_t len, uint8_t hash_out[32])
{
    if (!bm || !hash_out || (!data && len)) return GARAGE_EC_E_INVALID;
    BM_GUARD(bm->rpc_put_block_sealed(key32, data, len, hash_out));
}

int garage_bm_rpc_put_block_sealed_crc(garage_bm *bm, const uint8_t *key32, const uint8_t *data, size_t len,
                                       uint8_t crc_kind, uint8_t hash_out[32], uint32_t *crc_out)
{
    if (!bm || !hash_out || !crc_out || (!data && len) || crc_kind > GARAGE_EC_CRC_CRC32C) return GARAGE_EC_E_INVALID;
    BM_GUARD(bm->rpc_put_block_sealed(key32, data, len, hash_out, crc_kind, crc_out));
}

int garage_bm_rpc_get_block_opened(garage_bm *bm, const uint8_t hash[32], const uint8_t *key32, uint8_t *out, size_t cap,
                                   size_t *out_len)
{
    if (!bm || !hash || !key32 || !out || !out_len) return GARAGE_EC_E_INVALID;
    BM_GUARD(bm->rpc_get_block_opened(to_hash(hash), key32, out, cap, out_len));
}

void garage_bm_get_sealed_metrics(garage_bm *bm, garage_bm_sealed_metrics *o)
{
    if (!bm || !o) return;
    o->sealed_puts = bm->sealed_puts;
    o->sealed_batches = bm->sealed_batches;
    o->opened_gets = bm->opened_gets;
    o->opened_auth_failures = bm->opened_auth_failures;
    o->opened_fallbacks = bm->opened_fallbacks;
    o->seal_call_us = bm->seal_call_us;
    o->open_call_us = bm->open_call_us;
}

int garage_bm_rpc_get_block_range_opened(garage_bm *bm, const uint8_t hash[32], const uint8_t *key32, uint32_t offset,
                                         uint32_t len, uint8_t *out, size_t cap, size_t *out_len)
{
    if (!bm || !hash || !key32 || !out_len || (!out && len)) return GARAGE_EC_E_INVALID;
    BM_GUARD(bm->rpc_get_block_range_opened(to_hash(hash), key32, offset, len, out, cap, out_len));
}

int garage_bm_rpc_put_block_resealed(garage_bm *bm, const garage_bm_piece *pieces, int n_pieces, const uint8_t *src_key32,
                                     const uint8_t *dst_key32, uint8_t hash_out[32], uint32_t *stored_len_out)
{
    if (!bm || !pieces || !dst_key32 || !hash_out || n_pieces < 1 || n_pieces > GARAGE_BM_MAX_PIECES)
        return GARAGE_EC_E_INVALID;
    BM_GUARD(bm->rpc_put_block_resealed(pieces, n_pieces, src_key32, dst_key32, hash_out, stored_len_out));
}

int garage_bm_rpc_put_block_resealed_crc(garage_bm *bm, const garage_bm_piece *pieces, int n_pieces,
                                         const uint8_t *src_key32, const uint8_t *dst_key32, uint8_t crc_kind,
                                         uint8_t hash_out[32], uint32_t *stored_len_out, uint32_t *crc_out)
{
    if (!bm || !pieces || !dst_key32 || !hash_out || !crc_out || n_pieces < 1 || n_pieces > GARAGE_BM_MAX_PIECES ||
        crc_kind > GARAGE_EC_CRC_CRC32C)
        return GARAGE_EC_E_INVALID;
    BM_GUARD(bm->rpc_put_block_resealed(pieces, n_pieces, src_key32, dst_key32, hash_out, stored_len_out, crc_kind,
                                        crc_out));
}

void garage_bm_get_reseal_metrics(garage_bm *bm, garage_bm_reseal_metrics *o)
{
    if (!bm || !o) return;
    o->calls = bm->reseal_calls;
    o->batches = bm->reseal_batches;
    o->sources_gathered = bm->reseal_sources;
    o->bytes_read = bm->reseal_bytes_read;
    o->auth_failures = bm->reseal_auth_failures;
    o->fallbacks = bm->reseal_fallbacks;
    o->call_us = bm->reseal_us;
    o->reseal_call_us = bm->reseal_call_us;
}

void garage_bm_get_sealed_range_metrics(garage_bm *bm, garage_bm_sealed_range_metrics *o)
{
    if (!bm || !o) return;
    o->gets = bm->sealed_range_gets;
    o->degraded_gets = bm->sealed_range_degraded;
    o->bytes_read = bm->sealed_range_bytes_read;
    o->bytes_fetched = bm->sealed_range_bytes_fetched;
    o->auth_failures = bm->sealed_range_auth_failures;
    o->fallbacks = bm->sealed_range_fallbacks;
    o->call_us = bm->sealed_range_us;
    o->open_range_call_us = bm->sealed_range_call_us;
}

int garage_bm_rpc_get_block_range(garage_bm *bm, const uint8_t hash[32], uint32_t offset, uint32_t len, uint8_t *out,
                                  size_t cap, size_t *out_len)
{
    if (!bm || !hash || !out_len || (!out && len)) return GARAGE_EC_E_INVALID;
    BM_GUARD(bm->rpc_get_block_range(to_hash(hash), offset, len, out, cap, out_len));
}

int garage_bm_resync_block(garage_bm *bm, int node, const uint8_t hash[32])
{
    if (!bm || !hash || node < 0 || node >= (int)bm->nodes.size()) return GARAGE_EC_E_INVALID;
    BM_GUARD(bm->resync_block(node, to_hash(hash)));
}

int garage_bm_block_incref(garage_bm *bm, const uint8_t hash[32])
{
    if (!bm || !hash) return GARAGE_EC_E_INVALID;
    BM_GUARD((bm->block_incref(to_hash(hash)), GARAGE_BM_OK));
}

int garage_bm_block_decref(garage_bm *bm, const uint8_t hash[32])
{
    if (!bm || !hash) return GARAGE_EC_E_INVALID;
    BM_GUARD((bm->block_decref(to_hash(hash)), GARAGE_BM_OK));
}

long long garage_bm_get_block_rc(garage_bm *bm, const uint8_t hash[32])
{
    if (!bm || !hash) return -1;
    BM_GUARD((long long)bm->get_block_rc(to_hash(hash)));
}

int garage_bm_resync_all(garage_bm *bm, int node, int workers, uint64_t *resynced)
{
    if (!bm || node < 0 || node >= (int)bm->nodes.size()) return GARAGE_EC_E_INVALID;
    BM_GUARD(bm->resync_all(node, workers, resynced));
}

int garage_bm_repair_enqueue_missing(garage_bm *bm, int node, uint64_t *enqueued)
{
    if (!bm || node < 0 || node >= (int)bm->nodes.size()) return GARAGE_EC_E_INVALID;
    BM_GUARD(bm->repair_enqueue_missing(node, enqueued));
}

int garage_bm_resync_step(garage_bm *bm, int node, int workers, size_t max_blocks, uint64_t *resynced, uint64_t *failed,
                          uint64_t *deferred, int64_t *wait_ms)
{
    if (!bm || node < 0 || node >= (int)bm->nodes.size() || workers < 1 || workers > 8) return GARAGE_EC_E_INVALID;
    BM_GUARD(bm->resync_step(node, workers, max_blocks, resynced, failed, deferred, wait_ms));
}

int garage_bm_list_resync_errors(garage_bm *bm, int node, garage_bm_resync_error *out, size_t cap, size_t *n)
{
    if (!bm || node < -1 || node >= (int)bm->nodes.size() || !n || (!out && cap)) return GARAGE_EC_E_INVALID;
    BM_GUARD(bm->list_resync_errors(node, out, cap, n));
}

int garage_bm_resync_retry_now(garage_bm *bm, int node, const uint8_t *hash32, uint64_t *n)
{
    if (!bm || node < 0 || node >= (int)bm->nodes.size()) return GARAGE_EC_E_INVALID;
    BM_GUARD(([&] {
        const Hash h = hash32 ? to_hash(hash32) : Hash{};
        return bm->resync_retry_now(node, hash32 ? &h : nullptr, n);
    }()));
}

int garage_bm_block_info(garage_bm *bm, const uint8_t hash[32], int check_tags, garage_bm_block_status *out)
{
    if (!bm || !hash || !out) return GARAGE_EC_E_INVALID;
    BM_GUARD(bm->block_info(to_hash(hash), check_tags != 0, out));
}

int garage_bm_debug_set_clock_ms(garage_bm *bm, uint64_t now_ms)
{
    if (!bm || now_ms > (uint64_t)INT64_MAX) return GARAGE_EC_E_INVALID;
    bm->debug_clock_ms.store((int64_t)now_ms);
    return GARAGE_BM_OK;
}

void garage_bm_get_resync_metrics(garage_bm *bm, garage_bm_resync_metrics *o)
{
    if (!bm || !o) return;
    uint64_t entries = 0;
    for (auto &n : bm->nodes) {
        std::lock_guard<std::mutex> lk(n->mu);
        entries += n->resync_errors.size();
    }
    o->resync_error_entries = entries;
    o->resync_deferred = bm->resync_deferred;
    o->resync_steps = bm->resync_steps;
    o->resync_retry_nows = bm->resync_retry_nows;
    o->resync_failed_bytes_read = bm->resync_failed_bytes_read;
}

int garage_bm_scrub(garage_bm *bm, int node, uint64_t *checked, uint64_t *corrupt)
{
    if (!bm || node < 0 || node >= (int)bm->nodes.size()) return GARAGE_EC_E_INVALID;
    BM_GUARD(bm->scrub(node, checked, corrupt));
}

int garage_bm_scrub_step(garage_bm *bm, int node, const uint8_t *cursor32, size_t max_shards, uint8_t cursor_out32[32],
                         int *finished, uint64_t *checked, uint64_t *corrupt)
{
    return bm_step(bm, node, cursor32, cursor_out32, [&](const Hash *cur, Hash *out) {
        return bm->scrub(node, checked, corrupt, cur, max_shards, out, finished);
    });
}

int garage_bm_deep_scrub_step(garage_bm *bm, int node, const uint8_t *cursor32, size_t max_blocks,
                              uint8_t cursor_out32[32], int *finished, uint64_t *checked, uint64_t *repaired)
{
    return bm_step(bm, node, cursor32, cursor_out32, [&](const Hash *cur, Hash *out) {
        return bm->deep_scrub_step(node, cur, max_blocks, out, finished, checked, repaired);
    });
}

int garage_bm_stripe_repair_step(garage_bm *bm, int node, const uint8_t *cursor32, size_t max_blocks, int min_missing,
                                 uint8_t cursor_out32[32], int *finished, uint64_t *repaired_blocks,
                                 uint64_t *rebuilt_shards)
{
    return bm_step(bm, node, cursor32, cursor_out32, [&](const Hash *cur, Hash *out) {
        return bm->stripe_repair_step(node, cur, max_blocks, min_missing, out, finished, repaired_blocks, rebuilt_shards);
    });
}

int garage_bm_convert_step(garage_bm *bm, int node, const uint8_t *cursor32, size_t max_blocks, uint8_t cursor_out32[32],
                           int *finished, uint64_t *converted)
{
    return bm_step(bm, node, cursor32, cursor_out32, [&](const Hash *cur, Hash *out) {
        return bm->convert_step(node, cur, max_blocks, out, finished, converted);
    });
}

int garage_bm_apply_layout(garage_bm *bm, const garage_bm_layout_spec *spec, uint64_t *version_out)
{
    if (!bm || !spec) return GARAGE_EC_E_INVALID;
    BM_GUARD(bm->apply_layout(spec, version_out));
}

int garage_bm_layout_sync_step(garage_bm *bm, int node, const uint8_t *cursor32, size_t max_blocks, uint8_t cursor_out32[32],
                               int *finished, uint64_t *moved)
{
    return bm_step(bm, node, cursor32, cursor_out32, [&](const Hash *cur, Hash *out) {
        return bm->layout_sync_step(node, cur, max_blocks, out, finished, moved);
    });
}

int garage_bm_layout_versions(garage_bm *bm, uint64_t *out, int cap)
{
    if (!bm || cap < 0 || (cap > 0 && !out)) return GARAGE_EC_E_INVALID;
    const auto ls = bm->layouts();
    for (int i = 0; i < (int)ls->v.size() && i < cap; i++) out[i] = garage_layout_version(ls->v[i].get());
    return (int)ls->v.size();
}

int garage_bm_debug_convert_stop_after(garage_bm *bm, long n_ops)
{
    if (!bm) return GARAGE_EC_E_INVALID;
    bm->convert_ops_left.store(n_ops < 0 ? -1 : n_ops);
    return GARAGE_BM_OK;
}

int garage_bm_bench(garage_bm *bm, int threads, int blocks_per_thread, uint32_t block_len, int mode, uint64_t seed,
                    double *gib_per_s, uint64_t *errors)
{
    if (!bm || (mode != 0 && mode != 1)) return GARAGE_EC_E_INVALID;
    BM_GUARD(bm->bench(threads, blocks_per_thread, block_len, mode, seed, gib_per_s, errors));
}

int garage_bm_set_node_up(garage_bm *bm, int node, int up)
{
    if (!bm || node < 0 || node >= (int)bm->nodes.size()) return GARAGE_EC_E_INVALID;
    std::lock_guard<std::mutex> lk(bm->nodes[node]->mu);
    bm->nodes[node]->up = up != 0;
    return GARAGE_BM_OK;
}

static int bm_corrupt(garage_bm *bm, int node, const uint8_t hash[32], size_t byte_off, int what)
{
    Node &nd = *bm->nodes[node];
    std::lock_guard<std::mutex> lk(nd.mu);
    return nd.store_corrupt(to_hash(hash), byte_off, what);
}

int garage_bm_corrupt_shard(garage_bm *bm, int node, const uint8_t hash[32], size_t byte_off)
{
    if (!bm || !hash || node < 0 || node >= (int)bm->nodes.size()) return GARAGE_EC_E_INVALID;
    BM_GUARD(bm_corrupt(bm, node, hash, byte_off, 0));
}

int garage_bm_corrupt_shard_header(garage_bm *bm, int node, const uint8_t hash[32], int what)
{
    if (!bm || !hash || node < 0 || node >= (int)bm->nodes.size() || (what != 1 && what != 2)) return GARAGE_EC_E_INVALID;
    BM_GUARD(bm_corrupt(bm, node, hash, 0, what));
}

// replace the shard stored on `node` with a VALID shard (correct tag, correct index) of other
// content -- the "stale shard / wrong shard written by an earlier bad resync" case that only the
// whole-block content hash can catch
int garage_bm_plant_stale_shard(garage_bm *bm, int node, const uint8_t hash[32])
{
    if (!bm || !hash || node < 0 || node >= (int)bm->nodes.size()) return GARAGE_EC_E_INVALID;
    try {
        Node &nd = *bm->nodes[node];
        std::lock_guard<std::mutex> lk(nd.mu);
        StoredShard sh;
        const Hash h = to_hash(hash);
        if (!nd.store_get(h, sh) || sh.bytes.empty()) return GARAGE_BM_E_MISSING_BLOCK;
        for (size_t i = 0; i < sh.bytes.size(); i += 97) sh.bytes[i] ^= 0x5a;
        garage_ec_shard_sum_host(sh.sum_kind, sh.bytes.data(), sh.bytes.size(), sh.sum.data());
        return nd.store_put(h, sh, sh.bytes.data(), sh.bytes.size()) ? GARAGE_BM_OK : GARAGE_BM_E_MESSAGE;
    } catch (...) {
        return GARAGE_EC_E_NOMEM;
    }
}

int garage_bm_set_node_readonly(garage_bm *bm, int node, int readonly)
{
    if (!bm || node < 0 || node >= (int)bm->nodes.size()) return GARAGE_EC_E_INVALID;
    Node &nd = *bm->nodes[node];
    std::lock_guard<std::mutex> lk(nd.mu);
    if (nd.dir.empty()) return GARAGE_BM_E_MESSAGE;  // only meaningful for the file store
    // works for root too (which ignores permission bits): the directory is moved aside and a plain
    // FILE takes its name, so every create / open below it fails with ENOTDIR
    const std::string saved = nd.dir + ".moved_aside";
    if (readonly) {
        if (::rename(nd.dir.c_str(), saved.c_str()) != 0) return GARAGE_BM_E_MESSAGE;
        FILE *f = fopen(nd.dir.c_str(), "wb");
        if (f) fclose(f);
        return f ? GARAGE_BM_OK : GARAGE_BM_E_MESSAGE;
    }
    ::remove(nd.dir.c_str());
    return ::rename(saved.c_str(), nd.dir.c_str()) == 0 ? GARAGE_BM_OK : GARAGE_BM_E_MESSAGE;
}

int garage_bm_drop_shard(garage_bm *bm, int node, const uint8_t hash[32])
{
    if (!bm || !hash || node < 0 || node >= (int)bm->nodes.size()) return GARAGE_EC_E_INVALID;
    Node &nd = *bm->nodes[node];
    std::lock_guard<std::mutex> lk(nd.mu);
    if (nd.store_erase(to_hash(hash))) {
        bm->delete_counter++;
        return GARAGE_BM_OK;
    }
    return GARAGE_BM_E_MISSING_BLOCK;
}

int garage_bm_node_shard_index(garage_bm *bm, int node, const uint8_t hash[32])
{
    if (!bm || !hash || node < 0 || node >= (int)bm->nodes.size()) return -1;
    try {
        Node &nd = *bm->nodes[node];
        std::lock_guard<std::mutex> lk(nd.mu);
        StoredShard sh;
        return nd.store_get(to_hash(hash), sh) ? sh.index : -1;
    } catch (...) {
        return -1;
    }
}

int garage_bm_storage_nodes_of(garage_bm *bm, const uint8_t hash[32], int *nodes_out)
{
    if (!bm || !hash || !nodes_out) return GARAGE_EC_E_INVALID;
    bm->storage_nodes_of(to_hash(hash), nodes_out);
    return GARAGE_BM_OK;
}

void garage_bm_get_metrics(garage_bm *bm, garage_bm_metrics *o)
{
    if (!bm || !o) return;
    memset(o, 0, sizeof(*o));
    o->bytes_written = bm->bytes_written;
    o->bytes_read = bm->bytes_read;
    o->corruption_counter = bm->corruption_counter;
    o->resync_counter = bm->resync_counter;
    o->resync_error_counter = bm->resync_error_counter;
    o->resync_recv_counter = bm->resync_recv_counter;
    o->delete_counter = bm->delete_counter;
    o->put_calls = bm->put_calls;
    for (const auto &g : bm->groups) {
        o->put_batches += g->enc_batcher ? g->enc_batcher->batches() : 0;
        o->reconstruct_batches += g->rec_batcher ? g->rec_batcher->batches() : 0;
    }
    o->reconstruct_calls = bm->reconstruct_calls;
    o->scrub_shards_checked = bm->scrub_checked;
    o->scrub_corruptions = bm->scrub_corrupt;
    o->encode_call_us = bm->enc_gpu_us;
    o->reconstruct_call_us = bm->rec_gpu_us;
    o->corrupt_data_errors = bm->corrupt_data_errors;
    o->write_errors = bm->write_errors;
    o->resync_shards_read = bm->resync_shards_read;
    o->resync_bytes_read = bm->resync_bytes_read;
    o->resync_bytes_fetched = bm->resync_bytes_fetched;
    o->convert_blocks = bm->convert_blocks;
    o->convert_bytes_read = bm->convert_bytes_read;
    o->convert_bytes_written = bm->convert_bytes_written;
    o->convert_errors = bm->convert_errors;
    o->convert_call_us = bm->convert_call_us;
    o->legacy_gets = bm->legacy_gets;
    o->legacy_deleted = bm->legacy_deleted;
    o->layout_shards_copied = bm->layout_shards_copied;
    o->layout_shards_rebuilt = bm->layout_shards_rebuilt;
    o->layout_bytes_read = bm->layout_bytes_read;
    o->layout_bytes_written = bm->layout_bytes_written;
    o->layout_deleted = bm->layout_deleted;
    o->layout_sync_errors = bm->layout_sync_errors;
    o->layout_bytes_fetched = bm->layout_bytes_fetched;
    o->layout_version = garage_layout_version(bm->layouts()->newest());
    uint64_t ql = 0;
    for (auto &n : bm->nodes) {
        std::lock_guard<std::mutex> lk(n->mu);
        ql += n->resync_queue.size();
    }
    o->resync_queue_length = ql;
    o->deep_scrub_blocks = bm->deep_blocks;
    o->deep_scrub_skipped = bm->deep_skipped;
    o->deep_scrub_parity_bad = bm->deep_parity_bad;
    o->deep_scrub_content_errors = bm->deep_content_errors;
    o->deep_check_call_us = bm->deep_check_us;
}

void garage_bm_get_range_metrics(garage_bm *bm, garage_bm_range_metrics *o)
{
    if (!bm || !o) return;
    o->range_gets = bm->range_gets;
    o->range_degraded = bm->range_degraded;
    o->range_bytes_read = bm->range_bytes_read;
    o->range_bytes_fetched = bm->range_bytes_fetched;
}

int garage_bm_set_data_dirs(garage_bm *bm, int node, const garage_bm_data_dir *dirs, int n)
{
    if (!bm || node < 0 || node >= (int)bm->nodes.size() || !drive_list_ok(dirs, n)) return GARAGE_EC_E_INVALID;
    BM_GUARD(bm->set_data_dirs(node, dirs, n));
}

int garage_bm_rebalance_step(garage_bm *bm, int node, const uint8_t *cursor32, size_t max_files, uint8_t cursor_out32[32],
                             int *finished, uint64_t *moved)
{
    return bm_step(bm, node, cursor32, cursor_out32, [&](const Hash *cur, Hash *out) {
        return bm->rebalance_step(node, cur, max_files, out, finished, moved);
    });
}

void garage_bm_get_drive_metrics(garage_bm *bm, garage_bm_drive_metrics *o)
{
    if (!bm || !o) return;
    o->rebalance_files_moved = bm->rebalance_files_moved;
    o->rebalance_bytes_moved = bm->rebalance_bytes_moved;
    o->rebalance_errors = bm->rebalance_errors;
    o->drive_marker_errors = bm->drive_marker_errors;
}

void garage_bm_get_salvage_metrics(garage_bm *bm, garage_bm_salvage_metrics *o)
{
    if (!bm || !o) return;
    o->salvage_attempts = bm->salvage_attempts;
    o->salvage_blocks = bm->salvage_blocks;
    o->salvage_failures = bm->salvage_failures;
    o->salvage_units_rebuilt = bm->salvage_units_rebuilt;
    o->salvage_quarantined_segments = bm->salvage_quarantined_segments;
    o->salvage_bytes_read = bm->salvage_bytes_read;
    o->salvage_call_us = bm->salvage_call_us;
}

void garage_bm_get_segment_repair_metrics(garage_bm *bm, garage_bm_segment_repair_metrics *o)
{
    if (!bm || !o) return;
    o->repairs = bm->segrep_repairs;
    o->units_rebuilt = bm->segrep_units_rebuilt;
    o->bytes_read = bm->segrep_bytes_read;
    o->bytes_fetched = bm->segrep_bytes_fetched;
    o->fallbacks = bm->segrep_fallbacks;
    o->call_us = bm->segrep_call_us;
}

void garage_bm_get_stripe_repair_metrics(garage_bm *bm, garage_bm_stripe_repair_metrics *o)
{
    if (!bm || !o) return;
    o->stripe_repairs = bm->stripe_repairs;
    o->stripe_repair_shards = bm->stripe_repair_shards;
    o->stripe_repair_bytes_read = bm->stripe_repair_bytes_read;
    o->stripe_repair_bytes_fetched = bm->stripe_repair_bytes_fetched;
    o->stripe_repair_bytes_written = bm->stripe_repair_bytes_written;
    o->stripe_repair_errors = bm->stripe_repair_errors;
    o->stripe_repair_call_us = bm->stripe_repair_call_us;
}

}  // extern "C"
