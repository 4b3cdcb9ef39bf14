// llm_b200/csrc/snapshot.cu -- session snapshots: InferenceSession::get_snapshot / from_snapshot (crates/llm-base/src/inference_session.rs:591-646)
// and the CLI's session files (binaries/llm-cli/src/snapshot.rs), for every native session (include/llm_b200.h: b200_snapshot).
//
// The cache leaves and enters HBM in the reference's byte layout (RefKvLayout, host.h).  K and LLaMA / GPT-NeoX / GPT-J's V are the native bytes;
// GPT-2 / MPT / BLOOM keep V by position in the reference and by channel here, so those chunks go through transpose_kernel.  Every byte moves
// through a StreamRing of pinned and device buffers: a chunk's download overlaps the host's copy or fwrite of the previous ones (and the other
// way round on a restore), and the host never holds more than the ring.
#include <stdio.h>
#include <string.h>
#include <unistd.h>

#include <algorithm>
#include <memory>
#include <vector>

#include "../../include/llm_b200.h"
#include "host.h"

namespace b200 {

namespace {

constexpr int RING = 4;                         // chunks in flight
constexpr size_t CHUNK = 8u << 20;              // bytes per ring slot
constexpr uint64_t ZBLOCK = 128u << 10;         // zstd's largest block, and the window the writer declares
constexpr int64_t MAX_BATCH = 65536;
constexpr int64_t N_THREADS_WRITTEN = 8;        // InferenceSessionConfig::n_threads's default; not a property of a GPU session
constexpr uint8_t ZSTD_MAGIC[4] = {0x28, 0xB5, 0x2F, 0xFD};

// dst[c][r] = src[r][c] for r < rows, c < cols; T is the element's bit pattern (uint16_t: f16, uint32_t: f32), so NaNs and signed zeros move
// unchanged.  One CTA of 64 threads moves one TILE x TILE tile (TILE = 8 VEC, VEC = 16 / sizeof(T) elements: 64 x 64 f16, 32 x 32 f32).
// Thread (a, b) loads the VEC x VEC micro-tile at source rows VEC a + k, columns VEC b .. as VEC 16-byte vectors, transposes it in registers and
// stores it as VEC vectors into the tile in shared memory, which is kept in destination order; then 8 threads per destination row move the
// tile's rows to HBM in 16-byte vectors.  Lanes: a = lane & 7, b = 4 warp + (lane >> 3).
// Shared memory: a 16-byte access is served in four phases of 8 lanes, and in both stages the 8 lanes of a phase touch the 8 different 16-byte
// columns of one tile row, i.e. 8 disjoint groups of 4 banks -- conflict-free without padding.  HBM: 4 (load) and 8 (store) lanes cover 64 and
// 128 contiguous bytes of a row, whole 32-byte sectors.  vec == false (an unaligned base or stride) and the ragged edges of the matrix take
// element accesses.
template <class T>
__global__ void __launch_bounds__(64) transpose_kernel(const T *__restrict__ src, int64_t sld, T *__restrict__ dst, int64_t dld, int rows, int cols,
                                                       bool vec) {
    constexpr int VEC = 16 / sizeof(T), TILE = 8 * VEC;
    __shared__ __align__(16) T tile[TILE][TILE];            // [destination row = source column][destination column = source row]
    union V { int4 v; T e[VEC]; };
    const int lane = threadIdx.x & 31, a = lane & 7, b = 4 * (threadIdx.x >> 5) + (lane >> 3);
    const int r0 = blockIdx.y * TILE, c0 = blockIdx.x * TILE;
    V m[VEC];
#pragma unroll
    for (int k = 0; k < VEC; k++) {
        const int r = r0 + VEC * a + k, c = c0 + VEC * b;
        const T *p = src + (int64_t)r * sld + c;
        if (vec && r < rows && c + VEC <= cols) m[k].v = __ldg((const int4 *)p);
        else {
#pragma unroll
            for (int i = 0; i < VEC; i++) m[k].e[i] = (r < rows && c + i < cols) ? p[i] : T(0);
        }
    }
#pragma unroll
    for (int k = 0; k < VEC; k++) {
        V o;
#pragma unroll
        for (int i = 0; i < VEC; i++) o.e[i] = m[i].e[k];
        *(int4 *)&tile[VEC * b + k][VEC * a] = o.v;
    }
    __syncthreads();
    const int q = threadIdx.x & 7, r = r0 + VEC * q;
    for (int j = threadIdx.x >> 3; j < TILE && c0 + j < cols; j += 8) {
        V o;
        o.v = *(const int4 *)&tile[j][VEC * q];
        T *p = dst + (int64_t)(c0 + j) * dld + r;
        if (vec && r + VEC <= rows) *(int4 *)p = o.v;
        else {
#pragma unroll
            for (int i = 0; i < VEC; i++) if (r + i < rows) p[i] = o.e[i];
        }
    }
}

void transpose(size_t es, const void *src, int64_t sld, void *dst, int64_t dld, int64_t rows, int64_t cols, cudaStream_t st) {
    B200_ASSERT((es == 2 || es == 4) && rows >= 0 && cols >= 0 && rows < INT32_MAX && cols < INT32_MAX);
    if (rows == 0 || cols == 0) return;
    const int64_t vec_n = 16 / (int64_t)es, tile = 8 * vec_n;
    const bool vec = ((uintptr_t)src & 15) == 0 && ((uintptr_t)dst & 15) == 0 && sld % vec_n == 0 && dld % vec_n == 0;
    const dim3 grid((unsigned)((cols + tile - 1) / tile), (unsigned)((rows + tile - 1) / tile));
    B200_ASSERT(grid.y <= 65535);
    if (es == 2) transpose_kernel<uint16_t><<<grid, 64, 0, st>>>((const uint16_t *)src, sld, (uint16_t *)dst, dld, (int)rows, (int)cols, vec);
    else transpose_kernel<uint32_t><<<grid, 64, 0, st>>>((const uint32_t *)src, sld, (uint32_t *)dst, dld, (int)rows, (int)cols, vec);
    B200_CHECK(cudaGetLastError());
}

size_t kv_type_bytes(int32_t variant) { return variant == 1 ? 4 : 2; }     // ModelKVMemoryType: 0 Float16, 1 Float32
uint64_t ref_bytes(const RefKvLayout &L, int64_t n_ctx, size_t es) { return (uint64_t)L.n_layer * n_ctx * L.ref_width * es; }

using Sink = std::function<bool(const void *, size_t)>;

// memory_k (which 0) / memory_v (1) in the reference's layout, handed to `sink` in order, then the reference's unused tail as zeros
bool stream_out(const SessionCore &S, const RefKvLayout &L, int which, StreamRing &ring, const Sink &sink) {
    const size_t es = S.kv_elem_bytes();
    const int64_t n_ctx = S.n_ctx, W = L.width;
    const char *base = (const char *)S.kv_at(which, 0);
    bool ok = true;
    int64_t c = 0;
    auto retire = [&](StreamRing::Slot &sl) { if (sl.busy) { StreamRing::wait(sl); ok = ok && sink(sl.h, sl.bytes); } };
    auto issue = [&](size_t bytes, const std::function<void(StreamRing::Slot &)> &enqueue) {
        StreamRing::Slot &sl = ring.at(c++);
        retire(sl);                                               // chunk c - RING, the oldest in flight: the sink sees the chunks in order
        enqueue(sl);
        sl.bytes = bytes;
        B200_CHECK(cudaEventRecord(sl.done, sl.st));
        sl.busy = true;
    };
    if (which == 1 && L.v_by_position) {                          // [layer][W][n_ctx] -> [layer][n_ctx][W], a run of positions per chunk
        const int64_t per = std::max<int64_t>(1, (int64_t)(CHUNK / (W * es)));
        for (int l = 0; l < L.n_layer && ok; l++)
            for (int64_t p0 = 0; p0 < n_ctx && ok; p0 += per) {
                const int64_t np = std::min(per, n_ctx - p0);
                issue((size_t)(np * W * es), [&](StreamRing::Slot &sl) {
                    transpose(es, base + ((size_t)l * W * n_ctx + p0) * es, n_ctx, sl.d, W, W, np, sl.st);
                    B200_CHECK(cudaMemcpyAsync(sl.h, sl.d, (size_t)(np * W * es), cudaMemcpyDeviceToHost, sl.st));
                });
            }
    } else {
        const size_t total = S.kv_bytes();
        for (size_t o = 0; o < total && ok; o += CHUNK) {
            const size_t n = std::min(CHUNK, total - o);
            issue(n, [&](StreamRing::Slot &sl) { B200_CHECK(cudaMemcpyAsync(sl.h, base + o, n, cudaMemcpyDeviceToHost, sl.st)); });
        }
    }
    for (int k = 0; k < RING; k++) retire(ring.at(c + k));
    uint64_t tail = ref_bytes(L, n_ctx, es) - S.kv_bytes();        // LLaMA with grouped-query attention
    if (tail) {
        const std::vector<char> zeros((size_t)std::min<uint64_t>(tail, CHUNK), 0);
        for (; tail && ok; tail -= std::min<uint64_t>(tail, CHUNK)) ok = sink(zeros.data(), (size_t)std::min<uint64_t>(tail, CHUNK));
    }
    return ok;
}

// the inverse: `src` supplies the reference's bytes of one tensor in order; the tail is read and dropped.  The caller drains the ring.
bool stream_in(SessionCore &S, const RefKvLayout &L, int which, StreamRing &ring, const SnapshotSource &src) {
    const size_t es = S.kv_elem_bytes();
    const int64_t n_ctx = S.n_ctx, W = L.width;
    char *base = (char *)S.kv_at(which, 0);
    int64_t c = 0;
    auto issue = [&](size_t bytes, const std::function<void(StreamRing::Slot &)> &enqueue) {
        StreamRing::Slot &sl = ring.at(c++);
        StreamRing::wait(sl);                                     // its previous chunk has left the pinned buffer
        if (!src(sl.h, bytes)) return false;
        enqueue(sl);
        B200_CHECK(cudaEventRecord(sl.done, sl.st));
        sl.busy = true;
        return true;
    };
    if (which == 1 && L.v_by_position) {
        const int64_t per = std::max<int64_t>(1, (int64_t)(CHUNK / (W * es)));
        for (int l = 0; l < L.n_layer; l++)
            for (int64_t p0 = 0; p0 < n_ctx; p0 += per) {
                const int64_t np = std::min(per, n_ctx - p0);
                if (!issue((size_t)(np * W * es), [&](StreamRing::Slot &sl) {
                        B200_CHECK(cudaMemcpyAsync(sl.d, sl.h, (size_t)(np * W * es), cudaMemcpyHostToDevice, sl.st));
                        transpose(es, sl.d, W, base + ((size_t)l * W * n_ctx + p0) * es, n_ctx, np, W, sl.st);
                    })) return false;
            }
    } else {
        const size_t total = S.kv_bytes();
        for (size_t o = 0; o < total; o += CHUNK) {
            const size_t n = std::min(CHUNK, total - o);
            if (!issue(n, [&](StreamRing::Slot &sl) { B200_CHECK(cudaMemcpyAsync(base + o, sl.h, n, cudaMemcpyHostToDevice, sl.st)); })) return false;
        }
    }
    for (uint64_t tail = ref_bytes(L, n_ctx, es) - S.kv_bytes(); tail;) {
        const size_t n = (size_t)std::min<uint64_t>(tail, CHUNK);
        if (!issue(n, [](StreamRing::Slot &) {})) return false;
        tail -= n;
    }
    return true;
}

// ---- the session file: bincode of InferenceSnapshotRef inside one zstd frame -----------------------------------------------------------------
// bincode 1.3.3's default options: little-endian fixed-width integers, usize as u64, a sequence as its u64 count and the elements
struct Bincode {
    std::vector<uint8_t> b;
    template <class V> void put(V v) { const uint8_t *p = (const uint8_t *)&v; b.insert(b.end(), p, p + sizeof(V)); }
    void bytes(const void *p, size_t n) { b.insert(b.end(), (const uint8_t *)p, (const uint8_t *)p + n); }
};

// One zstd frame of raw blocks around `total` content bytes: header descriptor 0xC0 (8-byte content size, not single-segment, no checksum, no
// dictionary), window descriptor 0x38 (2^17 = 128 KiB), then 128 KiB blocks with 3-byte headers, the last one flagged.  A single-segment frame
// would declare the whole content as its window, which decoders refuse above 2^27 bytes by default.
struct ZstdRawWriter {
    FILE *fp; uint64_t total, done = 0; bool ok = true;
    ZstdRawWriter(FILE *f, uint64_t t) : fp(f), total(t) {
        uint8_t h[14] = {ZSTD_MAGIC[0], ZSTD_MAGIC[1], ZSTD_MAGIC[2], ZSTD_MAGIC[3], 0xC0, 0x38};
        for (int i = 0; i < 8; i++) h[6 + i] = (uint8_t)(t >> (8 * i));
        ok = fwrite(h, 1, sizeof(h), fp) == sizeof(h);
    }
    bool put(const void *p, size_t n) {
        const uint8_t *c = (const uint8_t *)p;
        B200_ASSERT(n <= total - done);
        while (n && ok) {
            if (done % ZBLOCK == 0) {
                const uint64_t bs = std::min(ZBLOCK, total - done);
                const uint32_t h = (uint32_t)(bs << 3) | (done + bs == total ? 1u : 0u);       // block type 0: raw
                const uint8_t hb[3] = {(uint8_t)h, (uint8_t)(h >> 8), (uint8_t)(h >> 16)};
                ok = fwrite(hb, 1, 3, fp) == 3;
            }
            const size_t m = (size_t)std::min<uint64_t>(n, ZBLOCK - done % ZBLOCK);
            ok = ok && fwrite(c, 1, m, fp) == m;
            c += m; n -= m; done += m;
        }
        return ok;
    }
};

// One zstd frame whose blocks are raw or RLE, checked whole when opened (every block header is read, no payload); then the content is read at
// any offset.  No zstd decoder is built here: a compressed block is B200_ERR_SNAPSHOT_FORMAT.
struct ZstdReader {
    struct Block { uint64_t file_off, content_off, size; bool rle; uint8_t byte; };
    FILE *fp = nullptr;
    std::vector<Block> blocks;
    uint64_t content = 0;
    ~ZstdReader() { if (fp) fclose(fp); }

    int open(const char *path) {
        if (!(fp = fopen(path, "rb"))) return B200_ERR_IO;
        if (fseeko(fp, 0, SEEK_END)) return B200_ERR_IO;
        const uint64_t fsize = (uint64_t)ftello(fp);
        uint64_t off = 0;
        auto get = [&](void *d, size_t n) { if (n > fsize - off) return false; const bool r = !fseeko(fp, (off_t)off, SEEK_SET) && fread(d, 1, n, fp) == n; off += n; return r; };
        auto le = [&](uint64_t &v, int n) { uint8_t b[8]; if (!get(b, n)) return false; v = 0; for (int i = 0; i < n; i++) v |= (uint64_t)b[i] << (8 * i); return true; };
        uint8_t magic[4], fhd;
        if (!get(magic, 4) || memcmp(magic, ZSTD_MAGIC, 4) || !get(&fhd, 1) || (fhd & 0x08)) return B200_ERR_SNAPSHOT_FORMAT;   // bit 3: reserved
        const bool single = fhd & 0x20, checksum = fhd & 0x04;
        const int fcs_n = (fhd >> 6) ? 1 << (fhd >> 6) : single ? 1 : 0, did_n = (fhd & 3) == 3 ? 4 : (fhd & 3);
        uint64_t window = 0, did, fcs = 0, wd;
        if (!single) {
            if (!le(wd, 1)) return B200_ERR_SNAPSHOT_FORMAT;
            const uint64_t base = 1ull << (10 + (wd >> 3));
            window = base + base / 8 * (wd & 7);
        }
        if ((did_n && !le(did, did_n)) || (fcs_n && !le(fcs, fcs_n))) return B200_ERR_SNAPSHOT_FORMAT;
        if (fcs_n == 2) fcs += 256;
        if (single) window = fcs;
        const uint64_t max_block = std::min(window, ZBLOCK);
        for (bool last = false; !last;) {
            uint64_t h;
            if (!le(h, 3)) return B200_ERR_SNAPSHOT_FORMAT;
            last = h & 1;
            const int type = (int)(h >> 1) & 3;
            const uint64_t size = h >> 3;
            if (type > 1 || size > max_block) return B200_ERR_SNAPSHOT_FORMAT;       // 2: compressed, 3: reserved
            Block b{off, content, size, type == 1, 0};
            if (type == 1 ? !get(&b.byte, 1) : size > fsize - off) return B200_ERR_SNAPSHOT_FORMAT;
            if (type == 0) off += size;
            blocks.push_back(b);
            content += size;
        }
        if (checksum && 4 > fsize - off) return B200_ERR_SNAPSHOT_FORMAT;            // present, not verified
        if (checksum) off += 4;
        if ((fcs_n && fcs != content) || off != fsize) return B200_ERR_SNAPSHOT_FORMAT;   // another frame or stray bytes after this one
        return B200_OK;
    }
    bool read_at(uint64_t pos, void *dst, size_t n) {
        if (n > content - std::min(pos, content)) return false;
        size_t bi = std::upper_bound(blocks.begin(), blocks.end(), pos, [](uint64_t p, const Block &b) { return p < b.content_off; }) - blocks.begin() - 1;
        for (char *d = (char *)dst; n; bi++) {
            const Block &b = blocks[bi];
            const uint64_t in = pos - b.content_off;
            if (in >= b.size) continue;
            const size_t m = (size_t)std::min<uint64_t>(n, b.size - in);
            if (b.rle) memset(d, b.byte, m);
            else if (fseeko(fp, (off_t)(b.file_off + in), SEEK_SET) || fread(d, 1, m, fp) != m) return false;
            d += m; n -= m; pos += m;
        }
        return true;
    }
};

}  // namespace

int snapshot_read_file(const char *path, SnapshotFile &f, bool with_data) {
    if (!path) return B200_ERR_BAD_ARG;
    std::shared_ptr<ZstdReader> r = std::make_shared<ZstdReader>();
    if (const int rc = r->open(path)) return rc;
    uint64_t pos = 0, u;
    uint32_t kt, vt;
    auto rd = [&](void *d, size_t n) { const bool ok = r->read_at(pos, d, n); pos += n; return ok; };
    auto count = [&](uint64_t &n, uint64_t elem) { return rd(&n, 8) && n <= (r->content - pos) / elem; };   // an overrun is a format error
    b200_snapshot &h = f.h;
    memset(&h, 0, sizeof(h));
    uint64_t v[3];
    if (!rd(&u, 8) || !rd(&kt, 4) || !rd(&vt, 4) || !rd(v, 16) || kt > 1 || vt > 1) return B200_ERR_SNAPSHOT_FORMAT;   // enum variant 0 / 1
    h.npast = (int64_t)std::min<uint64_t>(u, INT64_MAX); h.memory_k_type = (int32_t)kt; h.memory_v_type = (int32_t)vt;
    h.n_batch = (int64_t)std::min<uint64_t>(v[0], INT64_MAX); h.n_threads = (int64_t)std::min<uint64_t>(v[1], INT64_MAX);
    uint64_t nt, nl, mk, mv;
    if (!count(nt, 4)) return B200_ERR_SNAPSHOT_FORMAT;
    if (with_data) { f.tokens.resize(nt); if (!rd(f.tokens.data(), nt * 4)) return B200_ERR_IO; } else pos += nt * 4;
    if (!count(nl, 4)) return B200_ERR_SNAPSHOT_FORMAT;
    if (with_data) { f.last_logits.resize(nl); if (!rd(f.last_logits.data(), nl * 4)) return B200_ERR_IO; } else pos += nl * 4;
    if (!count(mk, 1)) return B200_ERR_SNAPSHOT_FORMAT;
    const uint64_t k_off = pos;
    pos += mk;
    if (!count(mv, 1) || mv != r->content - pos) return B200_ERR_SNAPSHOT_FORMAT;            // nothing may follow memory_v
    const uint64_t v_off = pos;
    h.n_tokens = (int64_t)nt; h.tokens = f.tokens.data();
    h.n_logits = (int64_t)nl; h.last_logits = f.last_logits.data();
    h.memory_k_bytes = mk; h.memory_v_bytes = mv;
    f.reader = r;
    f.k = [r, p = k_off](void *d, size_t n) mutable { const bool ok = r->read_at(p, d, n); p += n; return ok; };
    f.v = [r, p = v_off](void *d, size_t n) mutable { const bool ok = r->read_at(p, d, n); p += n; return ok; };
    return B200_OK;
}

int snapshot_check(const b200_snapshot &h, int n_ctx, int n_vocab, const RefKvLayout &L) {
    if (h.memory_k_type < 0 || h.memory_k_type > 1 || h.memory_v_type != h.memory_k_type) return B200_ERR_BAD_ARG;
    const uint64_t want = ref_bytes(L, n_ctx, kv_type_bytes(h.memory_k_type));
    if (h.memory_k_bytes != want || h.memory_v_bytes != want) return B200_ERR_SNAPSHOT_SIZE_MISMATCH;      // inference_session.rs:624-631
    if (h.npast < 0 || h.npast > n_ctx || h.n_tokens != h.npast || h.n_logits != n_vocab || h.n_batch < 1 || h.n_batch > MAX_BATCH) return B200_ERR_BAD_ARG;
    if ((h.n_tokens && !h.tokens) || !h.last_logits) return B200_ERR_BAD_ARG;
    for (int64_t i = 0; i < h.n_tokens; i++) if (h.tokens[i] >= (uint32_t)n_vocab) return B200_ERR_BAD_ARG;
    return B200_OK;
}

// the host-side fields of a snapshot: the history and the last row (zeros before the first evaluate, as the reference's initial last_logits)
static void snapshot_rows(const SessionCore &S, const float *logits, uint32_t *tokens, float *last) {
    B200_CHECK(cudaStreamSynchronize(rt().stream));               // after the work queued on the backend stream, as read_kv
    if (S.n_past) B200_CHECK(cudaMemcpy(tokens, S.history.get(), (size_t)S.n_past * 4, cudaMemcpyDeviceToHost));
    if (S.last_n < 1) memset(last, 0, (size_t)S.n_vocab * 4);
    else B200_CHECK(cudaMemcpy(last, logits + (size_t)(S.last_n - 1) * S.n_vocab, (size_t)S.n_vocab * 4, cudaMemcpyDeviceToHost));
}

int SessionCore::get_snapshot(const RefKvLayout &L, const float *logits, b200_snapshot *snap) {
    if (!snap) return B200_ERR_BAD_ARG;
    const uint64_t mem = ref_bytes(L, n_ctx, kv_elem_bytes());
    const int set = !!snap->tokens + !!snap->last_logits + !!snap->memory_k + !!snap->memory_v;
    if (set && (set != 4 || snap->n_tokens != n_past || snap->n_logits != n_vocab || snap->memory_k_bytes != mem || snap->memory_v_bytes != mem))
        return B200_ERR_BAD_ARG;
    snap->npast = n_past;
    snap->memory_k_type = snap->memory_v_type = kv_type == T_F32 ? 1 : 0;
    snap->n_batch = n_batch; snap->n_threads = N_THREADS_WRITTEN;
    snap->n_tokens = n_past; snap->n_logits = n_vocab;
    snap->memory_k_bytes = snap->memory_v_bytes = mem;
    if (!set) return B200_OK;
    snapshot_rows(*this, logits, snap->tokens, snap->last_logits);
    StreamRing ring(RING, CHUNK, CHUNK);
    for (int which = 0; which < 2; which++) {
        char *out = (char *)(which ? snap->memory_v : snap->memory_k);
        stream_out(*this, L, which, ring, [&out](const void *p, size_t n) { memcpy(out, p, n); out += n; return true; });
    }
    return B200_OK;
}

int SessionCore::write_snapshot(const RefKvLayout &L, const float *logits, const char *path) {
    if (!path) return B200_ERR_BAD_ARG;
    const uint64_t mem = ref_bytes(L, n_ctx, kv_elem_bytes());
    std::vector<uint32_t> tokens((size_t)n_past);
    std::vector<float> last((size_t)n_vocab);
    snapshot_rows(*this, logits, tokens.data(), last.data());
    Bincode b;                                                     // InferenceSnapshotRef up to memory_k's length
    b.put<uint64_t>(n_past);
    b.put<uint32_t>(kv_type == T_F32 ? 1 : 0); b.put<uint32_t>(kv_type == T_F32 ? 1 : 0);
    b.put<uint64_t>(n_batch); b.put<uint64_t>(N_THREADS_WRITTEN);
    b.put<uint64_t>(tokens.size()); b.bytes(tokens.data(), tokens.size() * 4);
    b.put<uint64_t>(last.size()); b.bytes(last.data(), last.size() * 4);
    b.put<uint64_t>(mem);
    FILE *fp = fopen(path, "wb");
    if (!fp) return B200_ERR_IO;
    ZstdRawWriter z(fp, b.b.size() + mem + 8 + mem);
    bool ok = z.put(b.b.data(), b.b.size());
    {
        StreamRing ring(RING, CHUNK, CHUNK);
        const Sink sink = [&z](const void *p, size_t n) { return z.put(p, n); };
        ok = ok && stream_out(*this, L, 0, ring, sink);
        ok = ok && z.put(&mem, 8);
        ok = ok && stream_out(*this, L, 1, ring, sink);
    }
    ok = (fclose(fp) == 0) && ok && z.done == z.total;
    if (!ok) { unlink(path); return B200_ERR_IO; }                // no partial file
    return B200_OK;
}

int SessionCore::restore_snapshot(const RefKvLayout &L, float *logits, const b200_snapshot &h, const SnapshotSource &k, const SnapshotSource &v) {
    cudaStream_t st = rt().stream;
    {
        StreamRing ring(RING, CHUNK, CHUNK);
        ring.after(st);
        if (!stream_in(*this, L, 0, ring, k) || !stream_in(*this, L, 1, ring, v)) return B200_ERR_IO;
        ring.drain();
    }
    if (h.npast) B200_CHECK(cudaMemcpyAsync(history.get(), h.tokens, (size_t)h.npast * 4, cudaMemcpyHostToDevice, st));
    B200_CHECK(cudaMemcpyAsync(logits, h.last_logits, (size_t)n_vocab * 4, cudaMemcpyHostToDevice, st));
    B200_CHECK(cudaStreamSynchronize(st));
    // the decode graphs upload their device copy of n_past before the next step, as after a rewind (DecodeGraphCache::run)
    n_past = (int)h.npast;
    last_n = 1;
    return B200_OK;
}

}  // namespace b200

using namespace b200;

extern "C" {

int b200_snapshot_read_header(const char *path, b200_snapshot *snap) {
    if (!snap) return B200_ERR_BAD_ARG;
    SnapshotFile f;
    const int rc = snapshot_read_file(path, f, false);
    if (rc == B200_OK) { *snap = f.h; snap->tokens = nullptr; snap->last_logits = nullptr; }
    return rc;
}

int b200_op_transpose_device(int32_t elem_bytes, const void *d_src, int64_t src_ld, void *d_dst, int64_t dst_ld, int64_t rows, int64_t cols) {
    if ((elem_bytes != 2 && elem_bytes != 4) || !d_src || !d_dst || rows < 0 || cols < 0 || rows >= INT32_MAX || cols >= INT32_MAX ||
        src_ld < cols || dst_ld < rows || (rows + 8 * 16 / elem_bytes - 1) / (8 * 16 / elem_bytes) > 65535) return B200_ERR_BAD_ARG;
    rt().ensure_init();
    transpose((size_t)elem_bytes, d_src, src_ld, d_dst, dst_ld, rows, cols, rt().stream);
    return B200_OK;
}

}  // extern "C"
