// engine.cu — the host-buffer picture pipeline of libsvtav1_b200.so (include/svt_av1_b200.h, "picture engine").
//
// The picture-level entries of the other files take DEVICE pointers and a stream.  The reference's process loops
// (motion_estimation_kernel, dlf_kernel, cdef_kernel; SURVEY.md §8b "Batched entry" / "Memory ownership") own HOST
// pictures and call from many pipeline threads at once, one picture per call.  The engine is the piece in between,
// inside the product library so that a C host gets it by linking (VERDICT r1 item 8):
//   * a residency cache of the three padded luma planes of every picture that ME touches (as source or as reference),
//     keyed by (host object, picture number): a picture is uploaded once and then serves as reference for the pictures
//     that follow it (EbPaReferenceObject lifetime, EbPictureBufferDesc.c:65-78 layout);
//   * per-call slots (stream + device scratch/outputs + pinned staging) so N threads run N pictures at once;
//   * the deblock -> CDEF search -> strength decision -> CDEF apply chain of one picture with the
//     reconstruction resident on the device across the stages.
// What costs in this setting is not the GPU work of a picture but CUDA calls that take process-wide locks while ~20
// pipeline threads are inside the library — cudaHostRegister of the caller's buffers (4 ms each and it stalls every other thread), cudaMalloc (device
// synchronisation) and pageable cudaMemcpy (holds the context lock for the whole host copy).  So every buffer is
// allocated ONCE, when the first picture fixes the geometry (one device arena, one pinned arena), host pictures are
// packed into the slot's pinned staging with plain memcpy outside any CUDA lock, and each call makes ~10 short
// asynchronous CUDA calls and one stream wait.
// Every entry is synchronous for its caller (the reference's stage returns when its picture is done) and re-entrant.
// There is no CPU fallback: a CUDA failure is returned as SVT_B200_ERR_CUDA and the integration aborts the encode.
#include <algorithm>
#include <condition_variable>
#include <mutex>
#include <thread>
#include <vector>

#include "common.cuh"

using namespace svtb200;

namespace {

constexpr int kMeSlots = 8;       // concurrent ME pictures
constexpr int kFiltSlots = 8;     // concurrent deblock / CDEF pictures
constexpr int kPlaneEntries = 96; // resident ME pictures (3.3 MB each at 1080p, 13 MB at 2160p); >= kMeSlots * 9 so that
                                  // every in-flight picture can hold its source + 8 references at once (no deadlock)
constexpr size_t kLutBytes = 3 * 2 * 128; // the level table of svt_b200_lf_level_lut

inline size_t al256(size_t v) { return (v + 255) & ~(size_t)255; }

// The next piece of an arena: pieces start 256-byte aligned, in the order they are taken.
template <typename T = uint8_t>
T *carve(uint8_t *&p, size_t bytes) {
    T *r = reinterpret_cast<T *>(p);
    p += al256(bytes);
    return r;
}

struct PlaneEntry {
    const void *key = nullptr;
    uint64_t tag = 0;
    uint8_t *d[3] = {nullptr, nullptr, nullptr};
    cudaEvent_t ready = nullptr;
    int state = 0; // 0 free, 1 loading, 2 ready
    int users = 0;
    uint64_t stamp = 0;
};

struct MeSlot {
    bool busy = false;
    cudaStream_t st = nullptr;
    cudaEvent_t up_done = nullptr; // the staging buffer has been consumed by its upload
    bool up_pending = false;
    uint8_t *scratch = nullptr;
    SvtB200MeOutputs out = {};  // device; me_mv | me_cand | total_cand | rc_me_distortion are contiguous
    uint8_t *pin_up = nullptr;  // full | quarter | sixteenth of one picture
    int16_t *pin_mv = nullptr;  // pinned copies of the four contiguous outputs, laid out alike: one read-back
    uint8_t *pin_cand = nullptr, *pin_tot = nullptr;
    uint32_t *pin_rc = nullptr;
};

struct FiltSlot {
    bool busy = false;
    cudaStream_t st = nullptr;
    SvtB200Frame recon, out, source; // device pictures
    // device, in this order: the LR units take the whole region from `mi` on
    SvtB200DlfMi *mi = nullptr;
    uint8_t *pick = nullptr; // svt_b200_pick_filter_level's scratch
    uint8_t *lut = nullptr;  // the level table of the picked levels
    uint8_t *skip = nullptr;
    uint64_t *mse = nullptr;
    int8_t *idx = nullptr;                 // filter-block strength indices,
    SvtB200CdefDecision *dec = nullptr;    // then the decision: one read-back
    uint8_t *decide = nullptr;             // svt_b200_cdef_decide's scratch
    // pinned
    uint8_t *pin_a = nullptr;     // packed picture (reconstruction up / down)
    uint8_t *pin_b = nullptr;     // packed picture (source), or the LR boundary lines
    uint8_t *pin_small = nullptr; // skip map | mse | fb idx | decision; also stages the LR units and the level table
    int8_t *pin_idx = nullptr;
    SvtB200CdefDecision *pin_dec = nullptr;
    SvtB200DlfMi *pin_mi = nullptr; // the mode-info array
};

struct MeGeom {
    size_t nb[3] = {0, 0, 0}, entry = 0, n_sb = 0, scratch = 0;
    size_t b_sad = 0, b_hme = 0, b_mv = 0, b_cand = 0, b_tot = 0, b_rc = 0, dev = 0, out = 0;
    bool operator==(const MeGeom &o) const { return nb[0] == o.nb[0] && nb[1] == o.nb[1] && nb[2] == o.nb[2] && n_sb == o.n_sb; }
};

struct FiltGeom {
    int w = 0, h = 0, bd = 0, mi_rows = 0, mi_cols = 0;
    int sy = 0, sc = 0; // device strides (samples)
    size_t by = 0, bc = 0, frame = 0, packed = 0, mi = 0, skip = 0, mse = 0, nfb = 0, misc = 0, small = 0, idx = 0, decide = 0;
    bool same(int w_, int h_, int bd_) const { return w == w_ && h == h_ && bd == bd_; }
};

} // namespace

struct SvtB200Engine {
    int device = 0;
    std::mutex mu;
    std::condition_variable cv;
    uint64_t clock = 0;
    PlaneEntry planes[kPlaneEntries];
    MeSlot me[kMeSlots];
    FiltSlot filt[kFiltSlots];
    // geometry-bound memory, allocated once by the first picture of each kind
    std::mutex init_mu;
    bool me_ready = false, filt_ready = false;
    MeGeom mg;
    FiltGeom fg;
    uint8_t *me_dev = nullptr, *me_pin = nullptr, *filt_dev = nullptr, *filt_pin = nullptr;
    struct {
        std::atomic<uint64_t> me_pictures{0}, dlf_frames{0}, cdef_frames{0}, lr_frames{0}, me_plane_uploads{0}, me_plane_hits{0}, h2d_bytes{0},
            d2h_bytes{0}, pinned_bytes{0}, ns_slot_wait{0}, ns_plane_wait{0}, ns_issue{0}, ns_sync{0}, ns_host_copy{0};
    } stats;
};

namespace {

inline uint64_t now_ns() {
    timespec t;
    clock_gettime(CLOCK_MONOTONIC, &t);
    return (uint64_t)t.tv_sec * 1000000000ull + (uint64_t)t.tv_nsec;
}
struct Lap { // accumulates wall time into an engine counter
    std::atomic<uint64_t> &acc;
    uint64_t t0;
    explicit Lap(std::atomic<uint64_t> &a) : acc(a), t0(now_ns()) {}
    ~Lap() { acc += now_ns() - t0; }
};

// ENG_TRY(expr): return from the calling function when expr fails.  expr is either a CUDA runtime call, whose error
// becomes the thread's message here, or a status from the library's entries and the engine's helpers, which set their
// own message.
inline int eng_status(cudaError_t err, const char *expr, const char *file, int line) {
    if (err == cudaSuccess) return SVT_B200_OK;
    set_error("engine: %s failed: %s (%s:%d)", expr, cudaGetErrorString(err), file, line);
    return SVT_B200_ERR_CUDA;
}
inline int eng_status(int rc, const char *, const char *, int) { return rc; }
#define ENG_TRY(expr)                                                                                              \
    do {                                                                                                           \
        const int rc__ = eng_status((expr), #expr, __FILE__, __LINE__);                                            \
        if (rc__ != SVT_B200_OK) return rc__;                                                                      \
    } while (0)

template <typename Slot, int N>
Slot *acquire(SvtB200Engine *e, Slot (&pool)[N]) {
    Lap lap(e->stats.ns_slot_wait);
    std::unique_lock<std::mutex> lk(e->mu);
    for (;;) {
        for (int i = 0; i < N; i++)
            if (!pool[i].busy) {
                pool[i].busy = true;
                return &pool[i];
            }
        e->cv.wait(lk);
    }
}

cudaError_t timed_sync(SvtB200Engine *e, cudaStream_t st) {
    Lap lap(e->stats.ns_sync);
    return cudaStreamSynchronize(st);
}

size_t plane_bytes(const SvtB200Plane &g) { return (size_t)g.stride * (size_t)(g.height + 2 * g.origin_y); }

// The device arena and the pinned arena of one side: both or, after a failure, neither.
int alloc_arenas(SvtB200Engine *e, uint8_t **dev, size_t dev_bytes, uint8_t **pin, size_t pin_bytes) {
    ENG_TRY(cudaMalloc((void **)dev, dev_bytes));
    const cudaError_t err = cudaMallocHost((void **)pin, pin_bytes);
    if (err != cudaSuccess) {
        cudaFree(*dev);
        *dev = nullptr;
        set_error("engine: cudaMallocHost of %zu bytes failed: %s", pin_bytes, cudaGetErrorString(err));
        return SVT_B200_ERR_CUDA;
    }
    e->stats.pinned_bytes += pin_bytes;
    return SVT_B200_OK;
}

// ---- one-time allocation for the ME side --------------------------------------------------------------------------
int ensure_me(SvtB200Engine *e, const SvtB200MeParams *p) {
    MeGeom g;
    g.nb[0] = plane_bytes(p->full);
    g.nb[1] = plane_bytes(p->quarter);
    g.nb[2] = plane_bytes(p->sixteenth);
    g.n_sb = (size_t)((p->full.width + 63) / 64) * ((p->full.height + 63) / 64);
    std::lock_guard<std::mutex> lk(e->init_mu);
    if (e->me_ready) {
        if (e->mg == g) return SVT_B200_OK;
        set_error("engine: the ME picture geometry changed (one engine serves one sequence geometry)");
        return SVT_B200_ERR_UNSUPPORTED;
    }
    g.entry = al256(g.nb[0]) + al256(g.nb[1]) + al256(g.nb[2]);
    g.scratch = al256(svt_b200_me_scratch_bytes(p));
    g.b_sad = g.n_sb * 8 * 85 * 4;
    g.b_hme = g.n_sb * 8 * sizeof(SvtB200HmeResult);
    g.b_mv = g.n_sb * 85 * 7 * 4;
    g.b_cand = g.n_sb * 85 * 23;
    g.b_tot = g.n_sb * 85;
    g.b_rc = g.n_sb * 4;
    g.out = al256(g.b_mv) + al256(g.b_cand) + al256(g.b_tot) + al256(g.b_rc);
    g.dev = 2 * al256(g.b_sad) + al256(g.b_hme) + g.out;
    const size_t dev_total = (size_t)kPlaneEntries * g.entry + (size_t)kMeSlots * (g.scratch + g.dev);
    const size_t pin_total = (size_t)kMeSlots * (g.entry + g.out);
    ENG_TRY(alloc_arenas(e, &e->me_dev, dev_total, &e->me_pin, pin_total));
    uint8_t *d = e->me_dev, *h = e->me_pin;
    for (auto &c : e->planes)
        for (int i = 0; i < 3; i++) c.d[i] = carve(d, g.nb[i]);
    for (auto &s : e->me) {
        s.scratch = carve(d, g.scratch);
        s.out.best_sad = carve<uint32_t>(d, g.b_sad);
        s.out.best_mv = carve<uint32_t>(d, g.b_sad);
        s.out.hme = carve<SvtB200HmeResult>(d, g.b_hme);
        s.out.me_mv = carve<int16_t>(d, g.b_mv);
        s.out.me_cand = carve(d, g.b_cand);
        s.out.total_cand = carve(d, g.b_tot);
        s.out.rc_me_distortion = carve<uint32_t>(d, g.b_rc);
        s.pin_up = carve(h, g.entry);
        s.pin_mv = carve<int16_t>(h, g.b_mv);
        s.pin_cand = carve(h, g.b_cand);
        s.pin_tot = carve(h, g.b_tot);
        s.pin_rc = carve<uint32_t>(h, g.b_rc);
    }
    e->mg = g;
    e->me_ready = true;
    return SVT_B200_OK;
}

// ---- one-time allocation for the deblock / CDEF side ---------------------------------------------------------------
int ensure_filt(SvtB200Engine *e, int w, int h, int bd, int mi_rows, int mi_cols) {
    std::lock_guard<std::mutex> lk(e->init_mu);
    if (e->filt_ready) {
        if (e->fg.same(w, h, bd)) return SVT_B200_OK;
        set_error("engine: the picture geometry changed (one engine serves one sequence geometry)");
        return SVT_B200_ERR_UNSUPPORTED;
    }
    FiltGeom g;
    g.w = w, g.h = h, g.bd = bd, g.mi_rows = mi_rows, g.mi_cols = mi_cols;
    const int bps = bd > 8 ? 2 : 1, cw = (w + 1) >> 1, ch = (h + 1) >> 1;
    g.sy = (w + 63) & ~63; // rows start 64-byte (8-bit) / 128-byte (16-bit) aligned: 128-bit vector access on every row
    g.sc = (cw + 63) & ~63;
    g.by = al256((size_t)g.sy * h * bps) + 256; // + slack between planes
    g.bc = al256((size_t)g.sc * ch * bps) + 256;
    g.frame = g.by + 2 * g.bc + 1024;
    g.packed = al256(((size_t)w * h + 2 * (size_t)cw * ch) * bps);
    g.mi = al256((size_t)mi_rows * mi_cols * sizeof(SvtB200DlfMi));
    g.nfb = (size_t)((mi_rows + 15) / 16) * ((mi_cols + 15) / 16);
    g.skip = al256((size_t)((mi_rows + 1) / 2) * ((((mi_cols + 1) / 2) + 15) & ~15));
    g.mse = al256(g.nfb * 2 * 64 * 8);
    g.idx = al256(g.nfb);
    g.decide = al256(g.nfb * (16 + 16 * 64) + 64); // any table size
    g.small = g.skip + g.mse + g.idx + al256(sizeof(SvtB200CdefDecision)) + g.decide;
    g.misc = g.mi + 4096 + g.small; // mode-info array | the level search's scratch and table | skip map ... decide scratch
    const size_t dev_total = (size_t)kFiltSlots * (3 * g.frame + g.misc);
    const size_t pin_total = (size_t)kFiltSlots * (2 * g.packed + g.small + g.mi);
    ENG_TRY(alloc_arenas(e, &e->filt_dev, dev_total, &e->filt_pin, pin_total));
    uint8_t *d = e->filt_dev, *hp = e->filt_pin;
    for (auto &s : e->filt) {
        for (SvtB200Frame *f : {&s.recon, &s.out, &s.source}) {
            uint8_t *b = carve(d, g.frame) + 512; // margin: the filters' vector loads may touch a few bytes before sample (0,0)
            f->y = b;
            f->cb = b + g.by;
            f->cr = b + g.by + g.bc;
            f->stride_y = g.sy;
            f->stride_c = g.sc;
            f->width = w;
            f->height = h;
            f->bit_depth = bd;
        }
        s.mi = carve<SvtB200DlfMi>(d, g.mi);
        s.pick = carve(d, 1024);
        s.lut = carve(d, 4096 - 1024);
        s.skip = carve(d, g.skip);
        s.mse = carve<uint64_t>(d, g.mse);
        s.idx = carve<int8_t>(d, g.idx);
        s.dec = carve<SvtB200CdefDecision>(d, sizeof(SvtB200CdefDecision));
        s.decide = carve(d, g.decide);
        s.pin_a = carve(hp, g.packed);
        s.pin_b = carve(hp, g.packed);
        s.pin_small = carve(hp, g.skip + g.mse); // the host uses neither the mse nor the decide-scratch part
        s.pin_idx = carve<int8_t>(hp, g.idx);
        s.pin_dec = carve<SvtB200CdefDecision>(hp, al256(sizeof(SvtB200CdefDecision)) + g.decide);
        s.pin_mi = carve<SvtB200DlfMi>(hp, g.mi);
    }
    e->fg = g;
    e->filt_ready = true;
    return SVT_B200_OK;
}

// memcpy split over kCopyThreads threads above kCopySplitBytes (see run_copies below); smaller copies stay on the
// calling thread (thread creation costs ~50 us)
constexpr size_t kCopySplitBytes = (size_t)4 << 20;
constexpr int kCopyThreads = 4;

void par_memcpy(void *dst, const void *src, size_t n) {
    if (n <= kCopySplitBytes) {
        memcpy(dst, src, n);
        return;
    }
    const size_t q = ((n / kCopyThreads) + 4095) & ~(size_t)4095;
    std::thread th[kCopyThreads - 1];
    for (int t = 1; t < kCopyThreads; t++) {
        const size_t o = q * t, len = o >= n ? 0 : std::min(q, n - o);
        th[t - 1] = std::thread([=] {
            if (len) memcpy((uint8_t *)dst + o, (const uint8_t *)src + o, len);
        });
    }
    memcpy(dst, src, std::min(q, n));
    for (auto &t : th) t.join();
}

// Every copy between pinned staging and the device goes through these two, which count the bytes they move.
void count_bytes(SvtB200Engine *e, cudaMemcpyKind kind, size_t n) {
    (kind == cudaMemcpyHostToDevice ? e->stats.h2d_bytes : e->stats.d2h_bytes) += n;
}
int copy_async(SvtB200Engine *e, void *dst, const void *src, size_t n, cudaMemcpyKind kind, cudaStream_t st) {
    ENG_TRY(cudaMemcpyAsync(dst, src, n, kind, st));
    count_bytes(e, kind, n);
    return SVT_B200_OK;
}
int copy_2d_async(SvtB200Engine *e, void *dst, size_t dpitch, const void *src, size_t spitch, size_t row, size_t rows,
                  cudaMemcpyKind kind, cudaStream_t st) {
    ENG_TRY(cudaMemcpy2DAsync(dst, dpitch, src, spitch, row, rows, kind, st));
    count_bytes(e, kind, row * rows);
    return SVT_B200_OK;
}

// The loader's part of plane_acquire: stage `pic` and upload it to `en` on the slot's stream (only the full plane when
// the decimations are derived on the device), then record `en`'s ready event.
int load_planes(SvtB200Engine *e, MeSlot *s, const SvtB200MeParams *p, const SvtB200HostMePicture *pic, int filtered_ds,
                PlaneEntry *en) {
    const MeGeom &g = e->mg;
    const bool gen = !pic->quarter || !pic->sixteenth; // decimations derived on the device
    if (s->up_pending) { // the staging buffer still feeds the previous upload of this call
        s->up_pending = false;
        ENG_TRY(cudaEventSynchronize(s->up_done));
    }
    size_t bytes = g.nb[0];
    {
        Lap lap(e->stats.ns_host_copy);
        par_memcpy(s->pin_up, pic->full, g.nb[0]);
        if (!gen) {
            memcpy(s->pin_up + al256(g.nb[0]), pic->quarter, g.nb[1]);
            memcpy(s->pin_up + al256(g.nb[0]) + al256(g.nb[1]), pic->sixteenth, g.nb[2]);
            bytes = al256(g.nb[0]) + al256(g.nb[1]) + g.nb[2]; // the three planes are laid out alike on both sides
        }
    }
    ENG_TRY(copy_async(e, en->d[0], s->pin_up, bytes, cudaMemcpyHostToDevice, s->st));
    ENG_TRY(cudaEventRecord(s->up_done, s->st));
    s->up_pending = true;
    if (gen) {
        const SvtB200MePlanes dp = {en->d[0], en->d[1], en->d[2]};
        ENG_TRY(svt_b200_me_downsample(&p->full, &p->quarter, &p->sixteenth, &dp, filtered_ds, s->st));
    }
    ENG_TRY(cudaEventRecord(en->ready, s->st));
    return SVT_B200_OK;
}

// A filter slot for the scope of one call.  A call that returns before its final stream wait may have left work on the
// slot's stream: the destructor waits for it before the slot can serve another call.
struct FiltLease {
    SvtB200Engine *e;
    FiltSlot *s;
    bool done = false; // the call's stream wait succeeded
    explicit FiltLease(SvtB200Engine *e_) : e(e_), s(acquire(e_, e_->filt)) {}
    ~FiltLease() {
        if (!done) cudaStreamSynchronize(s->st);
        {
            std::lock_guard<std::mutex> g(e->mu);
            s->busy = false;
        }
        e->cv.notify_all();
    }
};

// An ME slot and the plane entries its call made resident, for the scope of one call.  The entries are released after
// the stream wait: nothing of the picture may still read a plane when its entry is handed back.
struct MeLease {
    SvtB200Engine *e;
    MeSlot *s;
    PlaneEntry *ents[1 + SVT_B200_ME_LISTS * SVT_B200_ME_MAX_REFS] = {};
    int n_ent = 0;
    bool done = false; // the call's stream wait succeeded
    explicit MeLease(SvtB200Engine *e_) : e(e_), s(acquire(e_, e_->me)) {}
    ~MeLease() {
        if (!done) cudaStreamSynchronize(s->st);
        s->up_pending = false;
        {
            std::lock_guard<std::mutex> g(e->mu);
            for (int i = 0; i < n_ent; i++) ents[i]->users--;
            s->busy = false;
        }
        e->cv.notify_all();
    }
};

// Make the three planes of `pic` resident and ordered before later work on the slot's stream.  The lease holds the
// entry until it ends.
int plane_acquire(SvtB200Engine *e, MeLease &L, const SvtB200MeParams *p, const SvtB200HostMePicture *pic, int filtered_ds,
                  SvtB200MePlanes *out) {
    MeSlot *s = L.s;
    PlaneEntry *en = nullptr;
    bool loader = false;
    {
        std::unique_lock<std::mutex> lk(e->mu);
        for (;;) {
            PlaneEntry *victim = nullptr;
            for (auto &c : e->planes) {
                if (c.state && c.key == pic->key && c.tag == pic->tag) {
                    en = &c;
                    break;
                }
                if (c.users == 0 && c.state != 1 &&
                    (!victim || c.state < victim->state || (c.state == victim->state && c.stamp < victim->stamp)))
                    victim = &c;
            }
            if (en) {
                en->users++;
                {
                    Lap lap(e->stats.ns_plane_wait);
                    while (en->state == 1) e->cv.wait(lk);
                }
                if (en->state != 2) { // the loader failed
                    en->users--;
                    set_error("engine: upload of a reference picture failed in another thread");
                    return SVT_B200_ERR_CUDA;
                }
                e->stats.me_plane_hits++;
                break;
            }
            if (victim) {
                en = victim;
                en->key = pic->key;
                en->tag = pic->tag;
                en->state = 1;
                en->users = 1;
                loader = true;
                e->stats.me_plane_uploads++;
                break;
            }
            e->cv.wait(lk); // every entry is in use: wait for a picture to finish
        }
        en->stamp = ++e->clock;
    }
    if (loader) {
        const int rc = load_planes(e, s, p, pic, filtered_ds, en);
        {
            std::lock_guard<std::mutex> gl(e->mu);
            en->state = rc == SVT_B200_OK ? 2 : 0;
            if (rc != SVT_B200_OK) en->users--;
        }
        e->cv.notify_all();
        if (rc != SVT_B200_OK) return rc;
    }
    L.ents[L.n_ent++] = en;
    if (!loader) ENG_TRY(cudaStreamWaitEvent(s->st, en->ready, 0));
    *out = {en->d[0], en->d[1], en->d[2]};
    return SVT_B200_OK;
}

// The packed layout of a picture in pinned staging: tight rows, planes y, cb, cr one after another.  The host copies
// and the DMA copies of a picture both take it from here.
struct Packed {
    int bps = 0;              // bytes per sample
    int w[3], h[3];           // plane sizes in samples
    size_t row[3], off[3];    // bytes per packed row; where each plane starts in the staging buffer
    uint8_t *plane[3];        // the picture's planes
    size_t pitch[3];          // the picture's row pitches in bytes
    size_t bytes = 0;         // the whole packed picture
    explicit Packed(const SvtB200Frame *f) : bps(f->bit_depth > 8 ? 2 : 1) {
        for (int i = 0; i < 3; i++) {
            w[i] = i ? (f->width + 1) >> 1 : f->width;
            h[i] = i ? (f->height + 1) >> 1 : f->height;
            row[i] = (size_t)w[i] * bps;
            off[i] = bytes;
            bytes += row[i] * h[i];
            plane[i] = (uint8_t *)(i == 0 ? f->y : i == 1 ? f->cb : f->cr);
            pitch[i] = (size_t)(i ? f->stride_c : f->stride_y) * bps;
        }
    }
};

// host picture <-> packed pinned staging.  A 2160p 10-bit picture is 25 MB and one pipeline thread copies only a few
// GB/s (the picture pools of the encoder may be spread over both sockets of the host), so pictures above 4 MB are split
// by rows over four threads.
struct RowCopy {
    uint8_t *dst;
    const uint8_t *src;
    size_t dst_pitch, src_pitch, bytes;
    int rows;
};
void copy_rows(const RowCopy &c, int r0, int r1) {
    for (int y = r0; y < r1; y++) memcpy(c.dst + (size_t)y * c.dst_pitch, c.src + (size_t)y * c.src_pitch, c.bytes);
}
void run_copies(SvtB200Engine *e, const RowCopy (&c)[3]) {
    Lap lap(e->stats.ns_host_copy);
    size_t total = 0;
    for (const RowCopy &k : c) total += k.bytes * k.rows;
    const int nt = total > kCopySplitBytes ? kCopyThreads : 1;
    auto part = [&c, nt](int t) {
        for (const RowCopy &k : c) copy_rows(k, (int)((int64_t)k.rows * t / nt), (int)((int64_t)k.rows * (t + 1) / nt));
    };
    if (nt == 1) {
        part(0);
        return;
    }
    std::thread th[kCopyThreads - 1];
    for (int t = 1; t < nt; t++) th[t - 1] = std::thread(part, t);
    part(0);
    for (int t = 1; t < nt; t++) th[t - 1].join();
}
void pack_frame(SvtB200Engine *e, uint8_t *pin, const SvtB200Frame *f) {
    const Packed k(f);
    RowCopy c[3];
    for (int i = 0; i < 3; i++) c[i] = {pin + k.off[i], k.plane[i], k.row[i], k.pitch[i], k.row[i], k.h[i]};
    run_copies(e, c);
}
// planes: bit i set = write plane i of `f`
void unpack_frame(SvtB200Engine *e, const SvtB200Frame *f, const uint8_t *pin, unsigned planes = 7) {
    const Packed k(f);
    RowCopy c[3] = {};
    for (int i = 0; i < 3; i++)
        if (planes >> i & 1) c[i] = {k.plane[i], pin + k.off[i], k.pitch[i], k.row[i], k.row[i], k.h[i]};
    run_copies(e, c);
}
// packed pinned staging <-> device picture (three 2-D copies; both sides page-locked / device: pure DMA, asynchronous)
int copy_packed(SvtB200Engine *e, const SvtB200Frame *dev, uint8_t *pin, cudaMemcpyKind kind, cudaStream_t st) {
    const Packed k(dev);
    const bool up = kind == cudaMemcpyHostToDevice;
    for (int i = 0; i < 3; i++) {
        uint8_t *p = pin + k.off[i];
        ENG_TRY(copy_2d_async(e, up ? k.plane[i] : p, up ? k.pitch[i] : k.row[i], up ? p : k.plane[i], up ? k.row[i] : k.pitch[i],
                              k.row[i], k.h[i], kind, st));
    }
    return SVT_B200_OK;
}

struct DeviceGuard { // engine calls come from arbitrary pipeline threads: bind the engine's device for the call
    int prev = -1;
    explicit DeviceGuard(int dev) {
        cudaGetDevice(&prev);
        if (prev != dev)
            cudaSetDevice(dev);
        else
            prev = -1;
    }
    ~DeviceGuard() {
        if (prev >= 0) cudaSetDevice(prev);
    }
};

int create_streams(SvtB200Engine *e) {
    DeviceGuard g(e->device);
    for (auto &s : e->me) {
        ENG_TRY(cudaStreamCreateWithFlags(&s.st, cudaStreamNonBlocking));
        ENG_TRY(cudaEventCreateWithFlags(&s.up_done, cudaEventDisableTiming));
    }
    for (auto &s : e->filt) ENG_TRY(cudaStreamCreateWithFlags(&s.st, cudaStreamNonBlocking));
    for (auto &c : e->planes) ENG_TRY(cudaEventCreateWithFlags(&c.ready, cudaEventDisableTiming));
    return SVT_B200_OK;
}

} // namespace

extern "C" {

int svt_b200_engine_create(int device, SvtB200Engine **out) {
    if (!out) return SVT_B200_ERR_ARG;
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || device < 0 || device >= n) {
        set_error("svt_b200_engine_create: CUDA device %d not present (%d devices) - no CPU fallback", device, n);
        return SVT_B200_ERR_CUDA;
    }
    SvtB200Engine *e = new SvtB200Engine();
    e->device = device;
    if (const int rc = create_streams(e)) {
        svt_b200_engine_destroy(e);
        return rc;
    }
    *out = e;
    return SVT_B200_OK;
}

void svt_b200_engine_destroy(SvtB200Engine *e) {
    if (!e) return;
    DeviceGuard g(e->device);
    cudaDeviceSynchronize();
    for (auto &s : e->me) {
        if (s.st) cudaStreamDestroy(s.st);
        if (s.up_done) cudaEventDestroy(s.up_done);
    }
    for (auto &s : e->filt)
        if (s.st) cudaStreamDestroy(s.st);
    for (auto &c : e->planes)
        if (c.ready) cudaEventDestroy(c.ready);
    if (e->me_dev) cudaFree(e->me_dev);
    if (e->filt_dev) cudaFree(e->filt_dev);
    if (e->me_pin) cudaFreeHost(e->me_pin);
    if (e->filt_pin) cudaFreeHost(e->filt_pin);
    cudaGetLastError();
    delete e;
}

int svt_b200_engine_get_stats(SvtB200Engine *e, SvtB200EngineStats *out) {
    if (!e || !out) return SVT_B200_ERR_ARG;
    out->me_pictures = e->stats.me_pictures;
    out->dlf_frames = e->stats.dlf_frames;
    out->cdef_frames = e->stats.cdef_frames;
    out->lr_frames = e->stats.lr_frames;
    out->me_plane_uploads = e->stats.me_plane_uploads;
    out->me_plane_hits = e->stats.me_plane_hits;
    out->h2d_bytes = e->stats.h2d_bytes;
    out->d2h_bytes = e->stats.d2h_bytes;
    out->pinned_bytes = e->stats.pinned_bytes;
    out->ns_slot_wait = e->stats.ns_slot_wait;
    out->ns_plane_wait = e->stats.ns_plane_wait;
    out->ns_issue = e->stats.ns_issue;
    out->ns_sync = e->stats.ns_sync;
    out->ns_host_copy = e->stats.ns_host_copy;
    return SVT_B200_OK;
}

int svt_b200_engine_me_picture(SvtB200Engine *e, const SvtB200MeParams *p, const SvtB200HostMePicture *src,
                               const SvtB200HostMePicture refs[SVT_B200_ME_LISTS][SVT_B200_ME_MAX_REFS],
                               int32_t filtered_downsample, int16_t *me_mv, uint8_t *me_cand, uint8_t *total_cand,
                               uint32_t *rc_me_distortion) {
    if (!e || !p || !src || !refs || !me_mv || !me_cand || !total_cand || !rc_me_distortion || !src->full) {
        set_error("svt_b200_engine_me_picture: null argument");
        return SVT_B200_ERR_ARG;
    }
    for (int l = 0; l < p->num_lists; l++) {
        if (l >= SVT_B200_ME_LISTS || p->num_refs[l] > SVT_B200_ME_MAX_REFS) {
            set_error("svt_b200_engine_me_picture: more reference lists or references than SvtB200MeParams holds");
            return SVT_B200_ERR_ARG;
        }
        for (int r = 0; r < p->num_refs[l]; r++)
            if (!refs[l][r].full) {
                set_error("svt_b200_engine_me_picture: reference [%d][%d] has no planes", l, r);
                return SVT_B200_ERR_ARG;
            }
    }
    DeviceGuard dg(e->device);
    ENG_TRY(ensure_me(e, p));
    const MeGeom &g = e->mg;
    MeLease L(e);
    MeSlot *s = L.s;
    {
        Lap lap(e->stats.ns_issue);
        SvtB200MePlanes dsrc, drefs[SVT_B200_ME_LISTS][SVT_B200_ME_MAX_REFS] = {};
        ENG_TRY(plane_acquire(e, L, p, src, filtered_downsample, &dsrc));
        for (int l = 0; l < p->num_lists; l++)
            for (int r = 0; r < p->num_refs[l]; r++) ENG_TRY(plane_acquire(e, L, p, &refs[l][r], filtered_downsample, &drefs[l][r]));
        ENG_TRY(svt_b200_me_picture(p, &dsrc, drefs, &s->out, s->scratch, s->st));
        ENG_TRY(copy_async(e, s->pin_mv, s->out.me_mv, g.out, cudaMemcpyDeviceToHost, s->st));
    }
    ENG_TRY(timed_sync(e, s->st));
    L.done = true;
    Lap lap(e->stats.ns_host_copy);
    memcpy(me_mv, s->pin_mv, g.b_mv);
    memcpy(me_cand, s->pin_cand, g.b_cand);
    memcpy(total_cand, s->pin_tot, g.b_tot);
    memcpy(rc_me_distortion, s->pin_rc, g.b_rc);
    e->stats.me_pictures++;
    return SVT_B200_OK;
}

int svt_b200_engine_dlf_frame(SvtB200Engine *e, const SvtB200DlfParams *p, const SvtB200Frame *frame, const SvtB200DlfMi *mi) {
    if (!e || !p || !frame || !mi || p->mi_stride != p->mi_cols) {
        set_error("svt_b200_engine_dlf_frame: bad argument (mi_stride must equal mi_cols)");
        return SVT_B200_ERR_ARG;
    }
    DeviceGuard dg(e->device);
    ENG_TRY(ensure_filt(e, frame->width, frame->height, frame->bit_depth, p->mi_rows, p->mi_cols));
    const size_t b_mi = (size_t)p->mi_rows * p->mi_cols * sizeof(SvtB200DlfMi);
    if (b_mi > e->fg.mi) {
        set_error("svt_b200_engine_dlf_frame: mode-info array larger than the sequence geometry");
        return SVT_B200_ERR_ARG;
    }
    FiltLease L(e);
    FiltSlot *s = L.s;
    pack_frame(e, s->pin_a, frame);
    {
        Lap lap(e->stats.ns_host_copy);
        par_memcpy(s->pin_mi, mi, b_mi);
    }
    {
        Lap lap(e->stats.ns_issue);
        ENG_TRY(copy_async(e, s->mi, s->pin_mi, b_mi, cudaMemcpyHostToDevice, s->st));
        ENG_TRY(copy_packed(e, &s->recon, s->pin_a, cudaMemcpyHostToDevice, s->st));
        ENG_TRY(svt_b200_dlf_frame(p, &s->recon, s->mi, s->st));
        ENG_TRY(copy_packed(e, &s->recon, s->pin_a, cudaMemcpyDeviceToHost, s->st));
    }
    ENG_TRY(timed_sync(e, s->st));
    L.done = true;
    unpack_frame(e, frame, s->pin_a);
    e->stats.dlf_frames++;
    return SVT_B200_OK;
}

int svt_b200_engine_dlf_pick_frame(SvtB200Engine *e, const SvtB200LpfPickParams *pp, const SvtB200Frame *recon,
                                   const SvtB200Frame *source, const SvtB200DlfMi *mi, int32_t levels_out[4]) {
    if (!e || !pp || !recon || !source || !mi || !levels_out || pp->dlf.mi_stride != pp->dlf.mi_cols || recon->width != source->width ||
        recon->height != source->height || recon->bit_depth != source->bit_depth) {
        set_error("svt_b200_engine_dlf_pick_frame: bad argument");
        return SVT_B200_ERR_ARG;
    }
    DeviceGuard dg(e->device);
    ENG_TRY(ensure_filt(e, recon->width, recon->height, recon->bit_depth, pp->dlf.mi_rows, pp->dlf.mi_cols));
    const size_t b_mi = (size_t)pp->dlf.mi_rows * pp->dlf.mi_cols * sizeof(SvtB200DlfMi);
    if (b_mi > e->fg.mi) {
        set_error("svt_b200_engine_dlf_pick_frame: mode-info array larger than the sequence geometry");
        return SVT_B200_ERR_ARG;
    }
    FiltLease L(e);
    FiltSlot *s = L.s;
    pack_frame(e, s->pin_a, recon);
    {
        Lap lap(e->stats.ns_issue);
        ENG_TRY(copy_packed(e, &s->recon, s->pin_a, cudaMemcpyHostToDevice, s->st));
    }
    {
        Lap lap(e->stats.ns_host_copy);
        par_memcpy(s->pin_mi, mi, b_mi);
    }
    ENG_TRY(copy_async(e, s->mi, s->pin_mi, b_mi, cudaMemcpyHostToDevice, s->st));
    pack_frame(e, s->pin_b, source);
    ENG_TRY(copy_packed(e, &s->source, s->pin_b, cudaMemcpyHostToDevice, s->st));
    // every trial: one plane pass + SSE + plane restore on the device, one 8-byte read-back (the bisection is host logic)
    ENG_TRY(svt_b200_pick_filter_level(pp, &s->recon, &s->source, &s->out, s->mi, s->pick, levels_out, s->st));
    SvtB200DlfParams dp = pp->dlf;
    dp.sharpness = 0; // svt_av1_pick_filter_level sets lf->sharpness_level = 0 (EbDeblockingFilter.c:1202)
    dp.filter_level[0] = levels_out[0], dp.filter_level[1] = levels_out[1];
    dp.filter_level_u = levels_out[2], dp.filter_level_v = levels_out[3];
    dp.plane_start = 0, dp.plane_end = 3;
    svt_b200_lf_level_lut(&pp->init, levels_out, reinterpret_cast<uint8_t(*)[2][128]>(s->pin_small));
    {
        Lap lap(e->stats.ns_issue);
        ENG_TRY(copy_async(e, s->lut, s->pin_small, kLutBytes, cudaMemcpyHostToDevice, s->st));
        ENG_TRY(svt_b200_dlf_frame_lut(&dp, &s->recon, s->mi, s->lut, s->st));
        ENG_TRY(copy_packed(e, &s->recon, s->pin_a, cudaMemcpyDeviceToHost, s->st));
    }
    ENG_TRY(timed_sync(e, s->st));
    L.done = true;
    unpack_frame(e, recon, s->pin_a);
    e->stats.dlf_frames++;
    return SVT_B200_OK;
}

int svt_b200_engine_lr_frame(SvtB200Engine *e, const SvtB200LrFrameParams *p, const int32_t n_units[3], const SvtB200Frame *frame,
                             const SvtB200HostLrLines lines[3]) {
    if (!e || !p || !n_units || !frame || !lines) {
        set_error("svt_b200_engine_lr_frame: null argument");
        return SVT_B200_ERR_ARG;
    }
    DeviceGuard dg(e->device);
    ENG_TRY(ensure_filt(e, frame->width, frame->height, frame->bit_depth, (frame->height + 3) / 4, (frame->width + 3) / 4));
    const FiltGeom &g = e->fg;
    const Packed pk(frame);
    size_t b_units = 0;
    for (int i = 0; i < 3; i++) b_units += al256((size_t)std::max(n_units[i], 0) * sizeof(SvtB200LrUnit));
    // staging of the boundary lines: 4 rows per stripe boundary and plane
    size_t b_lines = 0;
    int nb[3], SH[3], off[3];
    unsigned restored = 0; // planes with restoration; the others stay as they are on the host, as in the reference
    for (int i = 0; i < 3; i++) {
        const int ss = i ? 1 : 0;
        SH[i] = 64 >> ss, off[i] = 8 >> ss;
        const int n_stripes = (pk.h[i] + off[i] + SH[i] - 1) / SH[i];
        nb[i] = p->plane[i].frame_restoration_type ? n_stripes - 1 : 0;
        if (p->plane[i].frame_restoration_type) restored |= 1u << i;
        b_lines += al256((size_t)nb[i] * 4 * pk.row[i]);
    }
    if (b_units + 256 > g.misc || b_lines > g.packed) {
        set_error("svt_b200_engine_lr_frame: unit / boundary-line arrays larger than the sequence geometry");
        return SVT_B200_ERR_ARG;
    }
    if (b_units > g.small) {
        set_error("svt_b200_engine_lr_frame: too many restoration units");
        return SVT_B200_ERR_ARG;
    }
    FiltLease L(e);
    FiltSlot *s = L.s;
    pack_frame(e, s->pin_a, frame);
    // units -> pin_small (host) -> the slot's device region from s->mi on, each plane's array 256-byte aligned
    SvtB200LrFrameParams dp = *p;
    size_t o = 0;
    for (int i = 0; i < 3; i++) {
        const size_t n = (size_t)std::max(n_units[i], 0) * sizeof(SvtB200LrUnit);
        if (n) memcpy(s->pin_small + o, p->plane[i].units, n);
        dp.plane[i].units = (const SvtB200LrUnit *)((uint8_t *)s->mi + o);
        o += al256(n);
    }
    // boundary lines: [boundary][row -2, -1, 0, +1 around the stripe edge][width], packed per plane in pin_b
    {
        Lap lap(e->stats.ns_host_copy);
        o = 0;
        for (int i = 0; i < 3; i++) {
            const size_t rb = pk.row[i], ls = (size_t)lines[i].stride * pk.bps;
            for (int b = 0; b < nb[i]; b++) {
                uint8_t *d = s->pin_b + o + (size_t)b * 4 * rb;
                const uint8_t *ab = (const uint8_t *)lines[i].above + (size_t)(2 * (b + 1)) * ls; // stripe b+1: rows y0-2, y0-1
                const uint8_t *be = (const uint8_t *)lines[i].below + (size_t)(2 * b) * ls;       // stripe b: rows y1, y1+1
                memcpy(d, ab, rb);
                memcpy(d + rb, ab + ls, rb);
                memcpy(d + 2 * rb, be, rb);
                memcpy(d + 3 * rb, be + ls, rb);
            }
            o += al256((size_t)nb[i] * 4 * rb);
        }
    }
    {
        Lap lap(e->stats.ns_issue);
        if (b_units) ENG_TRY(copy_async(e, s->mi, s->pin_small, b_units, cudaMemcpyHostToDevice, s->st));
        ENG_TRY(copy_packed(e, &s->recon, s->pin_a, cudaMemcpyHostToDevice, s->st));
        // scatter the boundary rows into a device picture that is only read at those rows (the deblocked context)
        const Packed ctx(&s->source);
        o = 0;
        for (int i = 0; i < 3; i++) {
            if (!nb[i]) continue;
            const size_t rb = pk.row[i];
            for (int k = 0; k < 4; k++) { // row B - 2 + k of every boundary B = (b + 1) * SH - off
                int rows = nb[i];
                if (nb[i] * SH[i] - off[i] - 2 + k >= pk.h[i]) rows--; // the last boundary's row lies below the plane
                if (rows <= 0) continue;
                ENG_TRY(copy_2d_async(e, ctx.plane[i] + (size_t)(SH[i] - off[i] - 2 + k) * ctx.pitch[i], ctx.pitch[i] * SH[i],
                                      s->pin_b + o + (size_t)k * rb, 4 * rb, rb, rows, cudaMemcpyHostToDevice, s->st));
            }
            o += al256((size_t)nb[i] * 4 * rb);
        }
        ENG_TRY(svt_b200_lr_frame(&dp, &s->recon, &s->source, &s->out, s->st));
        ENG_TRY(copy_packed(e, &s->out, s->pin_a, cudaMemcpyDeviceToHost, s->st));
    }
    ENG_TRY(timed_sync(e, s->st));
    L.done = true;
    unpack_frame(e, frame, s->pin_a, restored);
    e->stats.lr_frames++;
    return SVT_B200_OK;
}

// The CDEF stage of one picture, with the deblocking the DLF stage deferred (dlf != NULL) and the strength decision on
// the device (svt_b200_cdef_decide): one upload, deblocking, CDEF search, decision, CDEF apply, one download, ONE
// synchronisation - the reconstruction and the decision arrive together.  apply: 0 = search + decision only (EbCdefProcess.c:527-529: nobody reads the filtered picture).
int svt_b200_engine_dlf_cdef_frame_dev(SvtB200Engine *e, const SvtB200DlfParams *dlf, const SvtB200DlfMi *mi,
                                       const SvtB200CdefSearchParams *sp, const SvtB200CdefDecideParams *dp, int32_t damping,
                                       int32_t apply, const SvtB200Frame *recon, const SvtB200Frame *source, const uint8_t *skip8,
                                       int32_t skip_stride, SvtB200CdefDecision *decision, int8_t *fb_strength_idx) {
    if (!e || !sp || !dp || !recon || !source || !skip8 || !decision || !fb_strength_idx || recon->width != source->width ||
        recon->height != source->height || recon->bit_depth != source->bit_depth || (dlf && (!mi || dlf->mi_stride != dlf->mi_cols)) ||
        dp->mi_rows != sp->mi_rows || dp->mi_cols != sp->mi_cols || dp->n_strengths != sp->n_strengths) {
        set_error("svt_b200_engine_dlf_cdef_frame_dev: bad argument");
        return SVT_B200_ERR_ARG;
    }
    DeviceGuard dg(e->device);
    ENG_TRY(ensure_filt(e, recon->width, recon->height, recon->bit_depth, sp->mi_rows, sp->mi_cols));
    const FiltGeom &g = e->fg;
    const int nfb = ((sp->mi_rows + 15) / 16) * ((sp->mi_cols + 15) / 16);
    const size_t b_skip = (size_t)((sp->mi_rows + 1) / 2) * skip_stride;
    const size_t b_mi = dlf ? (size_t)dlf->mi_rows * dlf->mi_cols * sizeof(SvtB200DlfMi) : 0;
    if (al256(b_skip) > g.skip || (size_t)nfb > g.nfb || b_mi > g.mi) {
        set_error("svt_b200_engine_dlf_cdef_frame_dev: picture larger than the sequence geometry");
        return SVT_B200_ERR_ARG;
    }
    FiltLease L(e);
    FiltSlot *s = L.s;
    pack_frame(e, s->pin_a, recon);
    {
        Lap lap(e->stats.ns_host_copy);
        if (dlf) par_memcpy(s->pin_mi, mi, b_mi);
        memcpy(s->pin_small, skip8, b_skip);
    }
    {
        Lap lap(e->stats.ns_issue);
        if (dlf) ENG_TRY(copy_async(e, s->mi, s->pin_mi, b_mi, cudaMemcpyHostToDevice, s->st));
        ENG_TRY(copy_packed(e, &s->recon, s->pin_a, cudaMemcpyHostToDevice, s->st));
        if (dlf) ENG_TRY(svt_b200_dlf_frame(dlf, &s->recon, s->mi, s->st));
    }
    pack_frame(e, s->pin_b, source); // the host packs the source while the device receives and deblocks the reconstruction
    {
        Lap lap(e->stats.ns_issue);
        ENG_TRY(copy_async(e, s->skip, s->pin_small, b_skip, cudaMemcpyHostToDevice, s->st));
        ENG_TRY(copy_packed(e, &s->source, s->pin_b, cudaMemcpyHostToDevice, s->st));
        ENG_TRY(svt_b200_cdef_search(sp, &s->recon, &s->source, s->skip, skip_stride, s->mse, s->st));
        ENG_TRY(svt_b200_cdef_decide(dp, s->mse, s->skip, skip_stride, s->dec, s->idx, s->decide, s->st));
        if (apply) {
            ENG_TRY(svt_b200_cdef_apply_dev(sp->mi_rows, sp->mi_cols, damping, s->dec, &s->recon, &s->out, s->skip, skip_stride, s->idx,
                                            s->st));
            ENG_TRY(copy_packed(e, &s->out, s->pin_a, cudaMemcpyDeviceToHost, s->st));
        }
        // filter-block indices and the decision are adjacent on both sides: one copy
        ENG_TRY(copy_async(e, s->pin_idx, s->idx, g.idx + sizeof(SvtB200CdefDecision), cudaMemcpyDeviceToHost, s->st));
    }
    ENG_TRY(timed_sync(e, s->st));
    L.done = true;
    memcpy(fb_strength_idx, s->pin_idx, (size_t)nfb);
    memcpy(decision, s->pin_dec, sizeof(SvtB200CdefDecision));
    if (apply) unpack_frame(e, recon, s->pin_a);
    if (dlf) e->stats.dlf_frames++;
    e->stats.cdef_frames++;
    return SVT_B200_OK;
}

} // extern "C"
