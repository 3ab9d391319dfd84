// gate_host.cu -- C ABI (include/b200gate.h) and host planner of libb200gate.
//
// The planner turns the reference's chunk loop (noisereduce/spectralgate/base.py:167-226) into a
// table of independent (chunk, channel) units, sizes the device workspace, and launches
// k1_analyze -> k_rowfloor -> [k_smooth] -> k2_synthesize per batch of units on the caller's stream (the stationary
// gate's default synthesis kernel smooths the mask itself; k_smooth runs on the fallback paths).
#include "../../include/b200gate.h"
#include "gate_kernels_2k.cuh"
#include "gate_synth.cuh"
#include "gate_synth_2k.cuh"
#include "gate_dual.cuh"
#include "gate_peer.cuh"
#include "gate_generic.cuh"
#include "gate_convert.cuh"
#include "gate_adjoint.cuh"

#include <math.h>
#include <cmath>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <climits>
#include <condition_variable>
#include <functional>
#include <future>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

using namespace b200;

namespace {

const double kEps64 = 2.220446049250313e-16;       // np.finfo(np.float64).eps (spectralgate/utils.py:11)
const double kEps32 = 5.9604644775390625e-08;      // 2^-24, FP32 unit roundoff
const double kKappa = 16.0;                        // guard band: |dX| <= kappa * eps32 * ||frame pair||_2
thread_local std::string g_create_error;          // one handle per thread: a failed create reports through the calling thread
const char* const kTsOpen = "a torch stream is open on this handle (b200gate_tstream_finish first)";
constexpr int kSessSlots = 16;                     // depth of the per-row table upload ring (b200gate_tstream_push_rows)

}  // namespace

struct b200gate_handle {
    b200gate_params p{};
    std::string err;
    int num_sm = 132;
    int device = 0;
    int F = kF;
    // device tables
    float *d_wa = nullptr, *d_ws = nullptr, *d_invn = nullptr, *d_thr4 = nullptr, *d_gco = nullptr,
          *d_floor4 = nullptr, *d_ef = nullptr;
    float2* d_tw = nullptr;
    double *d_thr2_64 = nullptr, *d_wa64 = nullptr;
    double2* d_cs64 = nullptr;
    float ws_to_w = 0.f;
    float wa_max = 0.f;                            // max of the scaled analysis window (frame-energy bounds, gate_dual.cuh)
    unsigned* d_need_rowmax = nullptr;             // device flag raised by k1d_analyze when the top_db floor is reachable
    float2 *d_wa2 = nullptr, *d_ws2 = nullptr, *d_w2k = nullptr, *d_invn2 = nullptr;   // n_fft = 2048 family
    double sum_w = 0.0;
    std::vector<float> user_window;                // torch surface: torch.hann_window values
    float* d_tthr = nullptr;                       // torch surface: thresholds from xn, [tthr_units][FPad]
    int tthr_units = 0;
    bool have_thresh = false;
    double min_floor_amp = 0.0;                    // min_f 10^((thresh+top_db)/20): smallest |X| that lifts a row
    // b200gate_set_noise_threshold_rows: n_rec > 0 recordings' tables in one device buffer (have_thresh is then false):
    // thr4 | gco | floor4 as [n_rec][FPad] float, then thr2_64 as [n_rec][F] double (rec_tables())
    int n_rec = 0;
    void* d_rtab = nullptr;
    size_t rtab_bytes = 0;
    int range_mode = 0;                            // b200gate_set_range
    long long range_a = 0, range_b = 0;
    std::vector<double> thr, mean, sd;
    // general-geometry family (gate_generic.cuh)
    bool generic = false;
    int g_logN = 0;
    int g_M = 0, g_logM = 0;                       // Bluestein length for a non-power-of-two n_fft (0: radix-2 directly)
    double2 *d_gchirp = nullptr, *d_gbbr = nullptr;
    int g_W = 0;                                   // frame length: win_length (numpy surface) / n_fft (torch surface)
    double* d_gtthr = nullptr;                     // torch surface: thresholds from xn, [tthr_units][F]
    double *d_gwa = nullptr, *d_gws = nullptr, *d_gw2 = nullptr, *d_gthr = nullptr;
    double2* d_gcs = nullptr;
    // workspace
    char* d_ws_buf = nullptr;
    size_t ws_bytes = 0;
    void *d_in = nullptr, *d_out = nullptr;        // staging for host callers (kernel dtype)
    size_t in_bytes = 0, out_bytes = 0;
    void* d_raw = nullptr;                         // raw-dtype staging
    size_t raw_bytes = 0;
    Counters* d_cnt = nullptr;
    Counters* h_cnt = nullptr;                     // pinned: the run's exactness counters land here (stream-ordered copy)
    cudaEvent_t ev0 = nullptr, ev1 = nullptr, ev_done = nullptr;
    // statistics of a device-pointer run are resolved lazily (b200gate_get_stats): the run itself never blocks the host
    // torch surface: the masks of the last forward stay in the workspace so that the adjoint (= the same synthesis
    // with the same masks, TorchGate.backward) can reuse them -- b200gate_torch_apply_masks
    bool masks_valid = false, reuse_masks = false;
    long long masks_C = 0, masks_N = 0;
    std::vector<long long> masks_rows_n;           // ... of a b200gate_run_rows forward: its rows' lengths (else empty)
    // numpy surface: b200gate_set_mask_store's caller-owned buffer.  While it is set, b200gate_run carves the buffers
    // its kernels write the final masks to from it (every unit of the call) instead of from the workspace, and records
    // which run the store holds, so that b200gate_adjoint can check it is handed masks of its own geometry.
    void* mask_store = nullptr;
    int64_t mask_store_bytes = 0;
    bool keep_masks = false;                       // this b200gate_run keeps its masks in mask_store
    struct KeptRun { const void* store; long long C, N, a, b; int mode; size_t bytes; };
    std::vector<KeptRun> kept;                     // the stores filled by earlier runs (most recent last)
    bool stats_pending = false;
    size_t pend_batches = 0;
    std::vector<cudaEvent_t> group_ev;             // b200gate_run_sharded: one per channel group + 1
    std::vector<cudaEvent_t> stage_ev;             // 4 per batch: analysis start, analysis end, smoothing end, synthesis end
    std::vector<cudaEvent_t> pipe_ev;              // 4 per batch: input landed, compute done, output landed, seam copied
    cudaStream_t s_h2d = nullptr, s_d2h = nullptr; // pipelined host path
    void* hp_in[2] = {nullptr, nullptr};           // pinned staging slabs for pageable host rows (pipelined path)
    void* hp_out[2] = {nullptr, nullptr};
    size_t hp_in_bytes[2] = {0, 0}, hp_out_bytes[2] = {0, 0};
    int host_threads = 24;
    void* d_slab_in[2] = {nullptr, nullptr};       // caller-dtype slabs
    void* d_slab_out[2] = {nullptr, nullptr};
    size_t slab_in_bytes[2] = {0, 0}, slab_out_bytes[2] = {0, 0};
    b200gate_stats stats{};
    // streaming (b200gate_stream_*): a device window holding samples [s_lo, s_R) of every channel, row pitch s_cap
    bool s_open = false;
    int s_dtype = 0, s_is_device = -1;             // is_device of the stream's pushes (-1: none yet)
    long long s_C = 0, s_R = 0, s_E = 0, s_lo = 0; // samples received / returned; first sample in the window
    long long s_cap = 0, s_slice = 0, s_ocap = 0;  // window pitch, samples one slice appends at most, output pitch
    void *d_swin = nullptr, *d_sout = nullptr;
    size_t swin_bytes = 0, sout_bytes = 0;
    // TorchGate.stream() (b200gate_tstream_*): ts_B rows advancing together; ts_R samples received per row.  Frames
    // [0, ts_nA) have |X| and spectra, [0, ts_nM) the moving-mean mask, [0, ts_nS) the final mask; hops [2, ts_ha) have
    // been returned.  One device allocation holds the sample window [ts_lo, ts_R) (row pitch ts_cap) and the frame
    // rings of ts_ring frames (StreamWin); see b200gate_tstream_begin.
    bool ts_open = false;
    long long ts_B = 0, ts_R = 0, ts_lo = 0, ts_cap = 0, ts_slice = 0;
    long long ts_nA = 0, ts_nM = 0, ts_nS = 0, ts_ha = 2;
    int ts_ring = 0;
    void* d_ts = nullptr;
    float *d_ts_win = nullptr, *d_ts_mag = nullptr, *d_ts_m0 = nullptr, *d_ts_mask = nullptr;
    float2* d_ts_z = nullptr;
    double* d_ts_run = nullptr;
    // TorchGate.sessions() (b200gate_tstream_push_rows / _end_rows): every row holds its own session at its own position
    // (ts_row); each slice's per-row table (SessRow) is written into slot k of the pinned ring hp_sess and copied to slot
    // k of d_sess on the caller's stream, and ev_sess[k] marks that copy.  A slice waits for its slot's previous copy only,
    // so the host runs at most kSessSlots slices ahead of the device.  ts_mode: 0 until the first push, then 1 for the
    // lockstep calls or 2 for the per-row calls; a stream takes one kind only.
    struct TsRow { long long R = 0, lo = 0, nA = 0, nM = 0, nS = 0, ha = 2; };
    int ts_mode = 0;
    std::vector<TsRow> ts_row;
    std::vector<long long> ts_y0;                  // b200gate_tstream_push_rows: each row's output offset in the call
    SessRow* hp_sess = nullptr;
    size_t hp_sess_bytes = 0;
    SessRow* d_sess = nullptr;
    std::vector<cudaEvent_t> ev_sess;
    long long sess_slices = 0;
    // b200gate_run_rows: the call's unit table, written by the host into hp_units and copied to d_units on the call's
    // stream; ev_units marks that copy, so the next call can rewrite hp_units without waiting for the device
    UnitDesc* hp_units = nullptr;
    size_t hp_units_bytes = 0;
    void* d_units = nullptr;
    size_t units_bytes = 0;
    cudaEvent_t ev_units = nullptr;
    // debug taps
    long long dbg_chunk = -1, dbg_channel = -1;
    long long dbg_T = 0;
    float *d_dbg_spec = nullptr, *d_dbg_mask = nullptr;
    unsigned* d_dbg_bits = nullptr;
    size_t dbg_T_alloc = 0;
};

namespace {

int fail(b200gate_handle* h, int code, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    if (h) h->err = buf; else g_create_error = buf;
    return code;
}

#define CK(h, call)                                                                            \
    do {                                                                                       \
        cudaError_t e_ = (call);                                                               \
        if (e_ != cudaSuccess)                                                                 \
            return fail((h), B200GATE_ERR_CUDA, "%s failed: %s (%s:%d)", #call,               \
                        cudaGetErrorString(e_), __FILE__, __LINE__);                           \
    } while (0)

template <class T>
int upload(b200gate_handle* h, T** dptr, const std::vector<T>& v) {
    if (!*dptr) CK(h, cudaMalloc((void**)dptr, v.size() * sizeof(T)));
    CK(h, cudaMemcpy(*dptr, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice));
    return B200GATE_OK;
}

// one-call device scratch: freed on every return path
struct Scratch {
    void* p = nullptr;
    ~Scratch() { if (p) cudaFree(p); }
    Scratch() = default;
    Scratch(const Scratch&) = delete;
    Scratch& operator=(const Scratch&) = delete;
    cudaError_t alloc(size_t bytes) { return cudaMalloc(&p, bytes ? bytes : 1); }
    template <class T> T* as() const { return (T*)p; }
};

// A reduce_noise() call creates a handle, runs once and destroys it: its large device buffers (workspace, slabs, staging)
// would be cudaMalloc'ed and cudaFree'd every call (~15 ms together at config-2 sizes).  Destroyed handles leave them in a
// small process-wide cache instead (per device; bounded: B200GATE_DEVICE_CACHE_MB, default 4096, 0 disables), and ensure()
// looks there first.  Buffers enter the cache only after the device is idle (b200gate_destroy synchronises).
struct DevicePool {
    struct Item { void* p; size_t bytes; int dev; };
    std::mutex mu;
    std::vector<Item> items;
    size_t cached = 0;
    static size_t cap() {
        static const size_t c = [] {
            const char* e = getenv("B200GATE_DEVICE_CACHE_MB");
            return (size_t)(e ? std::max(0LL, atoll(e)) : 4096LL) << 20;
        }();
        return c;
    }
    void* take(size_t bytes, int dev, size_t* got) {
        std::lock_guard<std::mutex> lk(mu);
        size_t best = items.size();
        for (size_t i = 0; i < items.size(); ++i)
            if (items[i].dev == dev && items[i].bytes >= bytes && items[i].bytes <= bytes + bytes / 4 + (1 << 20) &&
                (best == items.size() || items[i].bytes < items[best].bytes))
                best = i;
        if (best == items.size()) return nullptr;
        void* p = items[best].p;
        *got = items[best].bytes;
        cached -= items[best].bytes;
        items.erase(items.begin() + (long)best);
        return p;
    }
    void give(void* p, size_t bytes, int dev) {            // the device must be idle with respect to p
        if (!p) return;
        {
            std::lock_guard<std::mutex> lk(mu);
            if (bytes >= (1 << 20) && cached + bytes <= cap() && items.size() < 16) {
                items.push_back(Item{p, bytes, dev});
                cached += bytes;
                return;
            }
        }
        cudaFree(p);
    }
    void drop_all(int dev) {                               // out of memory: give everything cached on this device back
        std::lock_guard<std::mutex> lk(mu);
        for (size_t i = items.size(); i-- > 0;)
            if (items[i].dev == dev) { cudaFree(items[i].p); cached -= items[i].bytes; items.erase(items.begin() + (long)i); }
    }
};
DevicePool g_device_pool;

int ensure(b200gate_handle* h, void** p, size_t* have, size_t need) {
    if (*have >= need) return B200GATE_OK;
    if (*p) cudaFree(*p);                                   // (synchronises: work still using the old buffer has finished)
    *p = nullptr;
    *have = 0;
    size_t got = 0;
    if (void* c = g_device_pool.take(need, h->device, &got)) {
        *p = c;
        *have = got;
        return B200GATE_OK;
    }
    cudaError_t e = cudaMalloc(p, need);
    if (e != cudaSuccess) {
        cudaGetLastError();
        g_device_pool.drop_all(h->device);
        e = cudaMalloc(p, need);
    }
    if (e != cudaSuccess) return fail(h, B200GATE_ERR_NOMEM, "cudaMalloc(%zu bytes) failed: %s", need, cudaGetErrorString(e));
    *have = need;
    return B200GATE_OK;
}

// Tables that depend only on the geometry: windows, twiddles, overlap-add norm, edge factors.
int build_static_tables_2k(b200gate_handle* h) {
    const int N = kN2, H = h->p.hop_length;
    std::vector<double> w(N);
    double sw = 0.0;
    for (int n = 0; n < N; ++n) {
        w[n] = 0.5 - 0.5 * cos(2.0 * M_PI * (double)n / (double)N);
        sw += w[n];
    }
    h->sum_w = sw;
    h->ws_to_w = (float)(1024.0 / sw);
    std::vector<float2> wa2(1024), ws2(1024), w2k(kF2), invn2(256), tw(32 * 32);
    for (int m = 0; m < 1024; ++m) {
        wa2[m] = make_float2((float)(w[2 * m] / sw), (float)(w[2 * m + 1] / sw));
        ws2[m] = make_float2((float)(w[2 * m] * sw / 1024.0), (float)(w[2 * m + 1] * sw / 1024.0));
    }
    for (int k = 0; k < kF2; ++k) {
        const long double th = M_PIl * (long double)k / 1024.0L;
        w2k[k] = make_float2((float)cosl(th), (float)(-sinl(th)));
    }
    for (int r = 0; r < H; ++r) {
        double sacc = 0.0;
        for (int i = 0; i * H + r < N; ++i) sacc += w[i * H + r] * w[i * H + r];
        const float v = (float)(sacc > 1e-10 ? 1.0 / sacc : 1.0);
        if (r & 1) invn2[r >> 1].y = v; else invn2[r >> 1].x = v;
    }
    for (int q = 0; q < 32; ++q)
        for (int l = 0; l < 32; ++l) {
            const long double th = 2.0L * M_PIl * (long double)(l * q) / 1024.0L;
            tw[q * 32 + l] = make_float2((float)cosl(th), (float)(-sinl(th)));
        }
    int rc;
    if ((rc = upload(h, &h->d_wa2, wa2))) return rc;
    if ((rc = upload(h, &h->d_ws2, ws2))) return rc;
    if ((rc = upload(h, &h->d_w2k, w2k))) return rc;
    if ((rc = upload(h, &h->d_invn2, invn2))) return rc;
    if ((rc = upload(h, &h->d_tw, tw))) return rc;
    return B200GATE_OK;
}

int build_static_tables(b200gate_handle* h) {
    if (h->p.n_fft == kN2) return build_static_tables_2k(h);
    const int N = h->p.n_fft, H = h->p.hop_length;
    std::vector<double> w(N);
    double sw = 0.0;
    for (int n = 0; n < N; ++n) {
        if ((int)h->user_window.size() == N) w[n] = (double)h->user_window[n];   // torch.hann_window (float32)
        else w[n] = 0.5 - 0.5 * cos(2.0 * M_PI * (double)n / (double)N);         // periodic Hann (scipy 'hann', fftbins)
        sw += w[n];
    }
    h->sum_w = sw;
    std::vector<float> wa(N), ws(N), invn(H);
    std::vector<double> wa64(N);
    for (int n = 0; n < N; ++n) {
        wa64[n] = w[n] / sw;
        wa[n] = (float)(w[n] / sw);
        ws[n] = (float)(w[n] * sw / (double)N);
    }
    h->ws_to_w = (float)((double)N / sw);
    h->wa_max = 0.f;
    for (int n = 0; n < N; ++n) h->wa_max = std::max(h->wa_max, (float)fabs(w[n] / sw) * (1.0f + 1e-6f));
    for (int r = 0; r < H; ++r) {
        double s = 0.0;
        for (int i = 0; i * H + r < N; ++i) s += w[i * H + r] * w[i * H + r];
        invn[r] = (float)(s > 1e-10 ? 1.0 / s : 1.0);
    }
    std::vector<float2> tw(32 * 32);
    for (int q = 0; q < 32; ++q)
        for (int l = 0; l < 32; ++l) {
            const long double th = 2.0L * M_PIl * (long double)(l * q) / 1024.0L;
            tw[q * 32 + l] = make_float2((float)cosl(th), (float)(-sinl(th)));
        }
    std::vector<double2> cs(N);
    for (int m = 0; m < N; ++m) {
        const long double th = 2.0L * M_PIl * (long double)m / (long double)N;
        cs[m] = make_double2((double)cosl(th), (double)sinl(th));
    }
    const int nf = h->p.n_grad_freq;
    std::vector<float> ef(kFPad, 0.f);
    for (int f = 0; f < kF; ++f) {
        long s = 0;
        for (int d = -nf; d <= nf; ++d)
            if (f - d >= 0 && f - d < kF) s += nf + 1 - abs(d);
        ef[f] = (float)((double)s / (double)((nf + 1) * (nf + 1)));
    }
    int rc;
    if ((rc = upload(h, &h->d_wa, wa))) return rc;
    if ((rc = upload(h, &h->d_ws, ws))) return rc;
    if ((rc = upload(h, &h->d_invn, invn))) return rc;
    if ((rc = upload(h, &h->d_tw, tw))) return rc;
    if ((rc = upload(h, &h->d_cs64, cs))) return rc;
    if ((rc = upload(h, &h->d_wa64, wa64))) return rc;
    if ((rc = upload(h, &h->d_ef, ef))) return rc;
    return B200GATE_OK;
}

// Tables that depend on the noise threshold (stationary.py:79-81), in the linear power domain:
// dB > thresh  <=>  |X| + eps > 10^(thresh/20)  <=>  |X|^2 > T_amp^2.
// One recording's rows from its thresholds thr[F] into thr4 / gco / floor4 [FPad] (pads left as they are) and t2 [F];
// returns min_floor_amp.  The single set and the per-recording tables both come from here, so they hold the same bits.
double threshold_rows(const b200gate_params& p, const double* thr, float* thr4, float* gco, float* floor4, double* t2) {
    double min_floor_amp = 0.0;
    for (int f = 0; f < kF; ++f) {
        double T = pow(10.0, thr[f] / 20.0) - kEps64;
        if (!(T > 0.0)) T = 0.0;
        double Tf = pow(10.0, (thr[f] + p.top_db) / 20.0) - kEps64;
        if (!(Tf > 0.0)) Tf = 0.0;
        t2[f] = T * T;
        if (f == 0 || Tf < min_floor_amp) min_floor_amp = Tf;
        thr4[f] = (float)(4.0 * T * T);
        gco[f] = (float)(8.0 * T * kKappa * kEps32 * (p.debug_guard_scale > 0 ? p.debug_guard_scale : 1));
        floor4[f] = (float)(4.0 * Tf * Tf);
    }
    return min_floor_amp;
}

int build_threshold_tables(b200gate_handle* h) {
    std::vector<float> thr4(kFPad, INFINITY), gco(kFPad, 0.f), floor4(kFPad, INFINITY);
    std::vector<double> t2(kF);
    h->min_floor_amp = threshold_rows(h->p, h->thr.data(), thr4.data(), gco.data(), floor4.data(), t2.data());
    int rc;
    if ((rc = upload(h, &h->d_thr4, thr4))) return rc;
    if ((rc = upload(h, &h->d_gco, gco))) return rc;
    if ((rc = upload(h, &h->d_floor4, floor4))) return rc;
    if ((rc = upload(h, &h->d_thr2_64, t2))) return rc;
    h->have_thresh = true;
    h->n_rec = 0;                                  // (a single set replaces per-recording thresholds)
    return B200GATE_OK;
}

// the device tables of per-recording thresholds (b200gate_set_noise_threshold_rows) in the layout of h->d_rtab
Tables rec_tables(const b200gate_handle* h, Tables tb) {
    const size_t R = (size_t)h->n_rec;
    float* f = (float*)h->d_rtab;
    tb.thr4 = f;
    tb.gco = f + R * kFPad;
    tb.floor4 = f + 2 * R * kFPad;
    tb.thr2_64 = (const double*)(f + 3 * R * kFPad);
    return tb;
}

Tables device_tables(const b200gate_handle* h) {
    Tables tb{};
    tb.wa = h->d_wa; tb.ws = h->d_ws; tb.tw = h->d_tw; tb.invn = h->d_invn;
    tb.thr4 = h->d_thr4; tb.gco = h->d_gco; tb.floor4 = h->d_floor4; tb.ef = h->d_ef;
    tb.thr2_64 = h->d_thr2_64; tb.wa64 = h->d_wa64; tb.cs64 = h->d_cs64;
    tb.ws_to_w = h->ws_to_w;
    return tb;
}

size_t dtype_size(int dtype) { return dtype == B200GATE_F32 ? 4 : dtype == B200GATE_I16 ? 2 : dtype == B200GATE_F64 ? 8 : 0; }

int grid_1d(long long n, int block, int cap) {
    long long g = (n + block - 1) / block;
    return (int)std::max(1LL, std::min<long long>(g, cap));
}

int generic_noise_stats_from_mean(b200gate_handle* h, const double* d_yn, long long n, cudaStream_t st);

// collapsed noise clip (float64, device) -> thresholds
int noise_stats_from_mean(b200gate_handle* h, const double* d_yn, long long n, cudaStream_t st) {
    if (h->generic) return generic_noise_stats_from_mean(h, d_yn, n, st);
    const int H = h->p.hop_length;
    const int Tn = (int)(n / H) + 1;                     // scipy: (n + 2*(W/2) - W)/H + 1
    Scratch s_db, s_res;
    CK(h, s_db.alloc((size_t)Tn * kF * sizeof(double)));
    CK(h, s_res.alloc(3 * kF * sizeof(double)));
    double *d_db = s_db.as<double>(), *d_res = s_res.as<double>();
    K0Args a{};
    a.yn = d_yn; a.n = n; a.H = H; a.Tn = Tn; a.wa64 = h->d_wa64; a.cs64 = h->d_cs64; a.eps = kEps64; a.db = d_db;
    B200_LAUNCH(k0_stft_db, dim3(Tn), dim3(256), kN * sizeof(double2), st, a);
    B200_LAUNCH(k0_stats, dim3(kF), dim3(256), 0, st, d_db, Tn, kF, h->p.top_db, h->p.std_ddof, h->p.n_std_thresh,
                d_res, d_res + kF, d_res + 2 * kF);
    CK(h, cudaGetLastError());
    std::vector<double> res(3 * kF);
    CK(h, cudaMemcpyAsync(res.data(), d_res, res.size() * sizeof(double), cudaMemcpyDeviceToHost, st));
    CK(h, cudaStreamSynchronize(st));
    h->mean.assign(res.begin(), res.begin() + kF);
    h->sd.assign(res.begin() + kF, res.begin() + 2 * kF);
    h->thr.assign(res.begin() + 2 * kF, res.end());
    return build_threshold_tables(h);
}

// ---- general-geometry family: tables, noise statistics ----------------------------------------------------------
int build_generic_tables(b200gate_handle* h) {
    const int N = h->p.n_fft, W = h->p.win_length;
    const bool torch_sem = h->p.surface != B200GATE_SURFACE_NUMPY;
    std::vector<double> w(W);
    double sw = 0.0;
    for (int n = 0; n < W; ++n) {
        if ((int)h->user_window.size() == W) w[n] = (double)h->user_window[n];             // torch.hann_window (float32)
        else if (torch_sem) w[n] = (double)(cosf((float)n * (float)(M_PI * 2.0 / W)) * -0.5f + 0.5f);
        else w[n] = 0.5 - 0.5 * cos(2.0 * M_PI * (double)n / (double)W);                  // scipy get_window('hann', W): periodic
        sw += w[n];
    }
    h->sum_w = sw;
    // numpy surface: frames of win_length samples, spectrum scaled by 1 / sum(w) (scaling='spectrum'), rfft pads at
    // the END.  torch surface (torch.stft, center=True): frames of n_fft samples under the window centre-padded
    // to n_fft, no scaling (torchgate.py:223-232).
    const int Wf = torch_sem ? N : W, left = torch_sem ? (N - W) / 2 : 0;
    h->g_W = Wf;
    std::vector<double> wa(Wf, 0.0), ws(Wf, 0.0), w2(Wf, 0.0);
    for (int n = 0; n < W; ++n) {
        wa[left + n] = torch_sem ? w[n] : w[n] / sw;
        ws[left + n] = torch_sem ? w[n] / (double)N : w[n] * sw / (double)N;               // irfft's 1/N (* sum(w) in scipy's istft)
        w2[left + n] = w[n] * w[n];
    }
    // transform tables: radix-2 twiddles of n_fft itself, or -- n_fft not a power of two -- Bluestein's chirp-z
    // through two length-M radix-2 transforms (M = 2^k >= 2 n_fft - 1)
    const int L = h->g_M ? h->g_M : N;
    std::vector<double2> cs(L);
    for (int m = 0; m < L; ++m) {
        const long double th = 2.0L * M_PIl * (long double)m / (long double)L;
        cs[m] = make_double2((double)cosl(th), (double)sinl(th));
    }
    int rc;
    if (h->g_M) {
        const int M = h->g_M, logM = h->g_logM;
        std::vector<double2> chirp(N);
        std::vector<long double> br(M, 0.0L), bi(M, 0.0L);
        for (int n = 0; n < N; ++n) {
            const long long q = ((long long)n * n) % (2LL * N);                  // n^2 mod 2N keeps the angle small
            const long double th = M_PIl * (long double)q / (long double)N;
            chirp[n] = make_double2((double)cosl(th), (double)(-sinl(th)));      // exp(-i pi n^2 / N)
            br[n] = cosl(th); bi[n] = sinl(th);                                  // conjugate chirp, circular
            if (n) { br[M - n] = br[n]; bi[M - n] = bi[n]; }
        }
        // forward FFT_M of the kernel in long double (iterative radix-2 DIT)
        for (int i = 0; i < M; ++i) {
            int r = 0;
            for (int b = 0; b < logM; ++b) r |= ((i >> b) & 1) << (logM - 1 - b);
            if (r > i) { std::swap(br[i], br[r]); std::swap(bi[i], bi[r]); }
        }
        for (int len = 2; len <= M; len <<= 1) {
            const int half = len >> 1;
            for (int blk = 0; blk < M; blk += len)
                for (int o = 0; o < half; ++o) {
                    const long double th = -2.0L * M_PIl * (long double)o / (long double)len;
                    const long double wr = cosl(th), wi = sinl(th);
                    const long double xr = br[blk + o], xi = bi[blk + o];
                    const long double yr = br[blk + o + half] * wr - bi[blk + o + half] * wi;
                    const long double yi = br[blk + o + half] * wi + bi[blk + o + half] * wr;
                    br[blk + o] = xr + yr; bi[blk + o] = xi + yi;
                    br[blk + o + half] = xr - yr; bi[blk + o + half] = xi - yi;
                }
        }
        std::vector<double2> bbr(M);
        for (int i = 0; i < M; ++i) {
            int r = 0;
            for (int b = 0; b < logM; ++b) r |= ((i >> b) & 1) << (logM - 1 - b);
            bbr[i] = make_double2((double)(br[r] / (long double)M), (double)(bi[r] / (long double)M));   // bit-reversed, 1/M folded in
        }
        if (h->d_gchirp) { cudaFree(h->d_gchirp); h->d_gchirp = nullptr; }
        if ((rc = upload(h, &h->d_gchirp, chirp))) return rc;
        if ((rc = upload(h, &h->d_gbbr, bbr))) return rc;
    }
    if ((rc = upload(h, &h->d_gwa, wa))) return rc;
    if ((rc = upload(h, &h->d_gws, ws))) return rc;
    if ((rc = upload(h, &h->d_gw2, w2))) return rc;
    if ((rc = upload(h, &h->d_gcs, cs))) return rc;
    return B200GATE_OK;
}

GTables generic_tables(const b200gate_handle* h) {
    GTables t{};
    t.wa = h->d_gwa; t.ws = h->d_gws; t.w2 = h->d_gw2; t.cs = h->d_gcs; t.chirp = h->d_gchirp; t.bbr = h->d_gbbr;
    return t;
}

GGeom generic_geom(const b200gate_handle* h, const Geom& g) {
    GGeom gg{};
    gg.g = g; gg.N = h->p.n_fft; gg.logN = h->g_logN; gg.W = h->g_W; gg.F = h->F; gg.out_len = 0;
    gg.M = h->g_M; gg.logM = h->g_logM;
    return gg;
}

int generic_threads(int N) { return N >= 512 ? 256 : std::max(32, (N / 2 + 31) / 32 * 32); }
int generic_fft_len(const b200gate_handle* h) { return h->g_M ? h->g_M : h->p.n_fft; }

int generic_noise_stats_from_mean(b200gate_handle* h, const double* d_yn, long long n, cudaStream_t st) {
    const int H = h->p.hop_length, W = h->p.win_length, N = h->p.n_fft, F = h->F;
    const long long Tn = (n + 2 * (W / 2) - W) / H + 1;
    if (Tn < 1 || Tn > 0x7fffffffLL) return fail(h, B200GATE_ERR_ARG, "noise clip length %lld unusable", n);
    Scratch s_X, s_db, s_res;
    CK(h, s_X.alloc((size_t)Tn * F * sizeof(double2)));
    CK(h, s_db.alloc((size_t)Tn * F * sizeof(double)));
    CK(h, s_res.alloc(3 * (size_t)F * sizeof(double)));
    double2* d_X = s_X.as<double2>();
    double *d_db = s_db.as<double>(), *d_res = s_res.as<double>();
    Geom g{};
    g.H = H; g.C = 1; g.T = (int)Tn; g.n_chunks = 1; g.n_total = n; g.step = n; g.pad = 0; g.Lp = n;
    g.in_stride = n; g.out_stride = n; g.u0 = 0; g.n_units = 1;
    GStftArgs<double> a{};
    a.gg = generic_geom(h, g); a.tb = generic_tables(h); a.x = d_yn; a.X = d_X;
    { auto kern_ = gk_stft<double>; B200_LAUNCH(kern_, dim3((unsigned)Tn, 1), dim3(generic_threads(generic_fft_len(h))), (size_t)generic_fft_len(h) * sizeof(double2), st, a); }
    B200_LAUNCH(gk_noise_db, dim3(grid_1d(Tn * F, 256, 1 << 16)), dim3(256), 0, st, (const double2*)d_X, (long long)Tn * F, kEps64, d_db);
    B200_LAUNCH(k0_stats, dim3(F), dim3(256), 0, st, d_db, (int)Tn, F, h->p.top_db, h->p.std_ddof, h->p.n_std_thresh,
                d_res, d_res + F, d_res + 2 * F);
    CK(h, cudaGetLastError());
    std::vector<double> res(3 * (size_t)F);
    CK(h, cudaMemcpyAsync(res.data(), d_res, res.size() * sizeof(double), cudaMemcpyDeviceToHost, st));
    CK(h, cudaStreamSynchronize(st));
    h->mean.assign(res.begin(), res.begin() + F);
    h->sd.assign(res.begin() + F, res.begin() + 2 * F);
    h->thr.assign(res.begin() + 2 * F, res.end());
    int rc = upload(h, &h->d_gthr, h->thr);
    if (rc) return rc;
    h->have_thresh = true;
    return B200GATE_OK;
}

template <typename Tin, typename Tacc>
void launch_channel_sum(const void* y, long long C, long long n, long long stride, void* acc, int init, cudaStream_t st) {
    auto kern = k0_channel_sum<Tin, Tacc>;
    B200_LAUNCH(kern, dim3(grid_1d(n, 256, 4096)), dim3(256), 0, st, (const Tin*)y, C, n, stride, (Tacc*)acc, init);
}

// Persistent host workers for the staging copies: a slab pipeline of ~50 slabs would otherwise create and join ~15 threads
// per slab and direction (~1 ms of a ~3 ms slab).  Workers sleep on a condition variable between jobs; one job at a time.
class HostWorkers {
public:
    // run work(id) for id in [0, nt) on nt - 1 pooled threads plus the caller
    void run(int nt, const std::function<void(int)>& work) {
        if (nt <= 1) { work(0); return; }
        std::unique_lock<std::mutex> job_lock(job_mu_);               // one job at a time (handles on several threads share the pool)
        {
            std::lock_guard<std::mutex> lk(mu_);
            while ((int)threads_.size() < nt - 1) {
                const int id = (int)threads_.size() + 1;
                threads_.emplace_back([this, id] { loop(id); });
            }
            work_ = &work;
            nt_ = nt;
            pending_ = nt - 1;
            ++generation_;
        }
        cv_.notify_all();
        work(0);
        std::unique_lock<std::mutex> lk(mu_);
        done_cv_.wait(lk, [this] { return pending_ == 0; });
        work_ = nullptr;
    }
    ~HostWorkers() {
        {
            std::lock_guard<std::mutex> lk(mu_);
            stop_ = true;
        }
        cv_.notify_all();
        for (auto& t : threads_) t.join();
    }

private:
    void loop(int id) {
        unsigned long long seen = 0;
        for (;;) {
            const std::function<void(int)>* w = nullptr;
            {
                std::unique_lock<std::mutex> lk(mu_);
                cv_.wait(lk, [&] { return stop_ || (generation_ != seen && id < nt_); });
                if (stop_) return;
                seen = generation_;
                w = work_;
            }
            (*w)(id);
            {
                std::lock_guard<std::mutex> lk(mu_);
                if (--pending_ == 0) done_cv_.notify_one();
            }
        }
    }
    std::mutex mu_, job_mu_;
    std::condition_variable cv_, done_cv_;
    std::vector<std::thread> threads_;
    const std::function<void(int)>* work_ = nullptr;
    int nt_ = 0, pending_ = 0;
    unsigned long long generation_ = 0;
    bool stop_ = false;
};
// pool 0: staging of pageable input rows; pool 1: copy-out of results into pageable rows (the two overlap in the slab pipeline)
HostWorkers& host_workers(int pool) {
    static HostWorkers* w[2] = {new HostWorkers(), new HostWorkers()};   // (never destroyed: no joins from static destructors at exit)
    return *w[pool & 1];
}

// device-resident (or staged) y -> running channel-order sum in acc
int channel_sum_impl(b200gate_handle* h, const void* y, int dtype, long long C, long long n, long long stride,
                     int is_device, void* acc, int init, cudaStream_t st) {
    const size_t es = dtype_size(dtype);
    const void* src = y;
    long long sstride = stride;
    Scratch tmp;
    if (!is_device && init) {
        // host rows: the channel-order sum is taken by the host workers (the same sequential additions in the same type, so
        // the same bits as k0_channel_sum) and only the n sums cross PCIe -- not C rows of pageable memory (64 x 600000 float32
        // through the driver's bounce buffer cost ~15 ms per reduce_noise() call)
        const size_t as = (dtype == B200GATE_F32) ? 4 : 8;
        std::vector<unsigned char> hacc((size_t)n * as);
        const long long blk = 8192;
        const long long n_blk = (n + blk - 1) / blk;
        const int nt = (int)std::max<long long>(1, std::min<long long>(std::min(h->host_threads, 32), n_blk));
        std::function<void(int)> work = [&](int id) {
            for (long long bix = id; bix < n_blk; bix += nt) {
                const long long i0 = bix * blk, i1 = std::min(n, i0 + blk);
                if (dtype == B200GATE_F32) {
                    float* a = (float*)hacc.data();
                    for (long long i = i0; i < i1; ++i) a[i] = 0.f;
                    for (long long c = 0; c < C; ++c) {
                        const float* r = (const float*)y + c * stride;
                        for (long long i = i0; i < i1; ++i) a[i] = a[i] + r[i];
                    }
                } else if (dtype == B200GATE_I16) {
                    double* a = (double*)hacc.data();
                    for (long long i = i0; i < i1; ++i) a[i] = 0.0;
                    for (long long c = 0; c < C; ++c) {
                        const short* r = (const short*)y + c * stride;
                        for (long long i = i0; i < i1; ++i) a[i] = a[i] + (double)r[i];
                    }
                } else {
                    double* a = (double*)hacc.data();
                    for (long long i = i0; i < i1; ++i) a[i] = 0.0;
                    for (long long c = 0; c < C; ++c) {
                        const double* r = (const double*)y + c * stride;
                        for (long long i = i0; i < i1; ++i) a[i] = a[i] + r[i];
                    }
                }
            }
        };
        host_workers(0).run(nt, work);
        CK(h, cudaMemcpyAsync(acc, hacc.data(), (size_t)n * as, cudaMemcpyHostToDevice, st));
        CK(h, cudaStreamSynchronize(st));                      // (hacc is freed on return)
        return B200GATE_OK;
    }
    if (!is_device) {
        CK(h, tmp.alloc((size_t)C * n * es));
        CK(h, cudaMemcpy2DAsync(tmp.p, (size_t)n * es, y, (size_t)stride * es, (size_t)n * es, (size_t)C,
                                cudaMemcpyHostToDevice, st));
        src = tmp.p;
        sstride = n;
    }
    if (dtype == B200GATE_F32) launch_channel_sum<float, float>(src, C, n, sstride, acc, init, st);
    else if (dtype == B200GATE_I16) launch_channel_sum<short, double>(src, C, n, sstride, acc, init, st);
    else launch_channel_sum<double, double>(src, C, n, sstride, acc, init, st);
    CK(h, cudaGetLastError());
    if (tmp.p) CK(h, cudaStreamSynchronize(st));          // the staging copy is freed on return
    return B200GATE_OK;
}

// run `stmt` with T bound to the kernels' sample type
#define B200_WITH_DTYPE(dt, ...)                                           \
    do {                                                                   \
        if ((dt) == B200GATE_I16) { using T = short; __VA_ARGS__; }        \
        else if ((dt) == B200GATE_F64) { using T = double; __VA_ARGS__; }  \
        else { using T = float; __VA_ARGS__; }                             \
    } while (0)

void launch_k1n(const Geom& g, const Tables& tb, const void* x, int kdt, float* mag, const DebugTap& dbg, int resident,
                cudaStream_t st, float2* zc = nullptr, int z_lo = 0, int z_hi = 0x7fffffff) {
    K1nArgs a1{};
    a1.g = g; a1.tb = tb; a1.x = x; a1.mag = mag; a1.dbg = dbg; a1.zcache = zc; a1.zpairs = (g.T + 1) / 2;
    a1.z_lo = z_lo; a1.z_hi = z_hi;
    long long want = (long long)resident * kWarps * 4;
    long long run = ((long long)g.n_units * g.T + want - 1) / want;
    run = std::max(8LL, std::min(64LL, run));
    run += run & 1;
    a1.run = (int)run;
    a1.n_runs = (g.T + a1.run - 1) / a1.run;
    B200_WITH_DTYPE(kdt, { auto kern_ = k1n_magnitude<8, T>;
        B200_LAUNCH(kern_, dim3(grid_1d((long long)g.n_units * a1.n_runs, kWarps, resident)), dim3(kThreads),
                    k1n_smem_floats() * 4, st, a1); });
}

// Binary-mask smoothing in byte lanes (k_smooth_packed, k2c_synthesize kMaskBits*): time sums up to (nt+1)^2 <= 196 per
// byte, biased first differences <= 31, at most 36 frequency taps; k_smooth_generic takes the rest.
static bool packed_smoothing_fits(int nf, int nt) { return nt + 1 <= 14 && 2 * nf + 1 <= 36; }

// k2c_synthesize kMaskBits*: a time-sum row keeps bin k at byte sm_pad + k with sm_pad a multiple of 16 (one 16-byte store
// per lane), so the tap window of bin 4i+j starts at byte 4 (i + sm_ws) + lead + j: the taps carry `lead` zero bytes first.
static void set_k2c_smoothing_taps(K2Args& a, int nf) {
    a.sm_pad = (nf + 15) & ~15;
    const int off = a.sm_pad - nf, lead = off & 3;
    a.sm_ws = off >> 2;
    const int words = (2 * nf + 1 + lead + 3) / 4;
    a.sm_ntw = words <= 4 ? 4 : words <= 7 ? 7 : words <= 9 ? 9 : kSynMaxTapWords;
    unsigned char tb8[4 * kSynMaxTapWords] = {0};
    for (int d = -nf; d <= nf; ++d) tb8[lead + d + nf] = (unsigned char)(nf + 1 - abs(d));
    memcpy(a.sm_taps, tb8, sizeof tb8);
}

// Stationary gate: the integer mask numerators of frames [sa.tf_lo, sa.tf_hi) from the decisions and row flags
// (k_smooth_packed where the byte lanes hold the filter, else k_smooth_generic).  `sa` carries the unit count, frames,
// filter extents, TT and the three buffers.
static void launch_stationary_numerators(const b200gate_handle* h, const SmoothArgs& sa, cudaStream_t st) {
    const int nf = sa.nf, nt = sa.nt, nu = sa.n_units, tf_lo = sa.tf_lo, tf_hi = sa.tf_hi;
    const int ntaps = 2 * nf + 1;
    if (packed_smoothing_fits(nf, nt)) {
        SmoothPArgs pa{};
        pa.n_units = nu; pa.T = sa.T; pa.nf = nf; pa.nt = nt; pa.tf_lo = tf_lo; pa.tf_hi = tf_hi;
        pa.bits = sa.bits; pa.rowflag = sa.rowflag; pa.num = sa.num;
        unsigned char tb8[36] = {0};
        for (int d = -nf; d <= nf; ++d) tb8[d + nf] = (unsigned char)(nf + 1 - abs(d));
        memcpy(pa.taps, tb8, 36);
        // strips: enough CTAs to fill the machine, long enough to amortise the 2 nt warm-up frames
        const int groups = (nu + kSmoothUnits - 1) / kSmoothUnits;
        int n_strips = std::max(1, std::min((tf_hi - tf_lo + 127) / 128, (h->num_sm * 4 + groups - 1) / groups));
        pa.strip = (tf_hi - tf_lo + n_strips - 1) / n_strips;
        pa.strip = (pa.strip + kSmoothBatch - 1) / kSmoothBatch * kSmoothBatch;     // frame pairs (2j, 2j+1) leave together
        n_strips = (tf_hi - tf_lo + pa.strip - 1) / pa.strip;
        const dim3 grid(n_strips, groups);
        if (ntaps <= 12) {
            B200_LAUNCH(k_smooth_packed<3>, grid, dim3(kSmoothThreads), smoothp_smem_bytes<3>(), st, pa);
        } else if (ntaps <= 24) {
            B200_LAUNCH(k_smooth_packed<6>, grid, dim3(kSmoothThreads), smoothp_smem_bytes<6>(), st, pa);
        } else {
            B200_LAUNCH(k_smooth_packed<9>, grid, dim3(kSmoothThreads), smoothp_smem_bytes<9>(), st, pa);
        }
    } else {
        const int tiles = (tf_hi - tf_lo + sa.TT - 1) / sa.TT;
        B200_LAUNCH(k_smooth_generic<>, dim3(tiles, nu), dim3(256), smooth_smem_bytes(sa.TT, nf, nt), st, sa);
    }
}

// Float-mask smoothing (non-stationary gate, TorchGate moving-mean gate): the box form for 1 <= nf <= 12 (k_smooth_box,
// compiled per nf), else the tap-loop streaming kernel, else (ring too large for shared memory) the tile kernel.
#define B200_SMOOTH_BOX_CASE(NF_) case NF_: { auto kern_ = k_smooth_box<NF_, ROWS, STREAM, SESS>; \
        if (set_attr) cudaFuncSetAttribute(kern_, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024); \
        else B200_LAUNCH(kern_, grid, dim3(sa.FPad / 4), smem, st, sa); } break;
template <bool ROWS = false, bool STREAM = false, bool SESS = false>
static void smooth_box_dispatch(const SmoothFArgs& sa, int nf, dim3 grid, size_t smem, cudaStream_t st, bool set_attr) {
    switch (nf) {
        B200_SMOOTH_BOX_CASE(1) B200_SMOOTH_BOX_CASE(2) B200_SMOOTH_BOX_CASE(3) B200_SMOOTH_BOX_CASE(4)
        B200_SMOOTH_BOX_CASE(5) B200_SMOOTH_BOX_CASE(6) B200_SMOOTH_BOX_CASE(7) B200_SMOOTH_BOX_CASE(8)
        B200_SMOOTH_BOX_CASE(9) B200_SMOOTH_BOX_CASE(10) B200_SMOOTH_BOX_CASE(11) B200_SMOOTH_BOX_CASE(12)
        default: break;
    }
}
// ROWS (b200gate_run_rows; sa.units set, tf_hi the largest of the batch) and STREAM (b200gate_tstream_*; sa.sw set;
// with SESS sa.rows set, tf_hi - tf_lo the largest span of a row): the two streaming kernels only -- false when the ring
// does not fit shared memory.
template <bool ROWS = false, bool STREAM = false, bool SESS = false>
static bool launch_smooth_float(SmoothFArgs sa, int nf, int nt, int tf_lo, int tf_hi, int nu, int path_flags, cudaStream_t st) {
    const bool box_ok = nf >= 1 && nf <= 12 && sa.FPad - sa.F >= 12 && smoothb_smem_bytes(sa.FPad, nt) <= 200 * 1024 &&
                        !(path_flags & 32) && !(path_flags & 128);
    if (box_ok) {
        sa.TT = 256;                        // frames per strip (2 nt warm-up rows each)
        const int strips = (tf_hi - tf_lo + sa.TT - 1) / sa.TT;
        smooth_box_dispatch<ROWS, STREAM, SESS>(sa, nf, dim3(strips, nu), smoothb_smem_bytes(sa.FPad, nt), st, false);
    } else if (smooths_smem_bytes(sa.FPad, nf, nt) <= 200 * 1024 && !(path_flags & 32)) {
        sa.TT = 256;
        const int strips = (tf_hi - tf_lo + sa.TT - 1) / sa.TT;
        auto kern_ = k_smooth_stream<ROWS, STREAM, SESS>;
        B200_LAUNCH(kern_, dim3(strips, nu), dim3(sa.FPad / 4), smooths_smem_bytes(sa.FPad, nf, nt), st, sa);
    } else if (ROWS || STREAM) {
        return false;
    } else {
        const int tiles = (tf_hi - tf_lo + sa.TT - 1) / sa.TT;
        B200_LAUNCH(k_smooth_f, dim3(tiles, nu), dim3(256), smoothf_smem_bytes(sa.TT, sa.FPad, nf), st, sa);
    }
    return true;
}

// k_iir_sigmoid may rebuild its forward sweep by the inverse recurrence (IirArgs::regen) only where the bound on the
// relative error of the follower S that this costs, 2.5 u (1-b)^(-2T) / b with u = 2^-53 (derived at k_iir_sigmoid),
// stays within 2^-24, the float32 rounding the stored forward sweep puts on S:  2 T ln(1/(1-b)) - ln b <= 29 ln 2 - ln 2.5.
// (Config 3, 48 kHz / n_fft 2048 / 600000-sample chunks: T = 1290, b = 0.00532 -> 19.00 of 19.19.)
static int iir_regen_ok(double b, int T, int path_flags) {
    if (path_flags & 64 || !(b < 0.5)) return 0;
    return 2.0 * (double)T * -log1p(-b) - log(b) <= 29.0 * log(2.0) - log(2.5) ? 1 : 0;
}

// Pageable host memory: cudaMemcpyAsync from / to it is neither asynchronous nor fast (the driver bounces it through a small
// pinned buffer at ~10 GB/s), and pinning a caller's 7 GB array in place costs a second (measured: cudaHostRegister 8.5 GB/s).
// The slab pipeline therefore stages pageable rows through its own pinned slabs with a handful of host threads
// (measured 60-70 GB/s with 8-16 threads), which keeps PCIe busy.
bool host_pointer_is_pinned(const void* p) {
#ifdef B200_CUSIM_BUILD
    (void)p;
    return false;                                  // simulator: exercise the staging path
#else
    cudaPointerAttributes at{};
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return at.type == cudaMemoryTypeHost || at.type == cudaMemoryTypeManaged;
#endif
}
void parallel_rows_copy(void* dst, size_t dpitch, const void* src, size_t spitch, size_t width, size_t rows, int nthreads,
                        int pool = 0) {
    if (rows == 0 || width == 0) return;
    // split every row into pieces of >= 1 MB so that few long rows still spread over all threads
    const size_t piece = std::max<size_t>(1 << 20, (width * rows / (size_t)std::max(1, nthreads) + 4095) / 4096 * 4096);
    const size_t per_row = (width + piece - 1) / piece;
    const size_t n_pieces = per_row * rows;
    const int nt = (int)std::min<size_t>((size_t)std::max(1, std::min(nthreads, 64)), n_pieces);
    std::function<void(int)> work = [&](int id) {
        for (size_t k = (size_t)id; k < n_pieces; k += (size_t)nt) {
            const size_t r = k / per_row, off = (k - r * per_row) * piece;
            memcpy((char*)dst + r * dpitch + off, (const char*)src + r * spitch + off, std::min(piece, width - off));
        }
    };
    host_workers(pool).run(nt, work);
}

// Pinned staging slabs are expensive to create (cudaMallocHost of 1 GB: ~0.2 s) and independent of the handle's parameters:
// they live in a small process-wide pool, borrowed for one run and returned (a handle is created per reduce_noise() call).
struct PinnedPool {
    std::mutex mu;
    std::vector<std::pair<void*, size_t>> free_list;
    std::vector<std::pair<void*, size_t>> leased;          // b200gate_host_alloc: sizes of the buffers callers hold
    // best fit, and never a buffer more than twice the request (a 7 GB result buffer must not end up as a 256 MB slab)
    void* take(size_t bytes, size_t* got) {
        {
            std::lock_guard<std::mutex> lk(mu);
            size_t best = free_list.size();
            for (size_t i = 0; i < free_list.size(); ++i)
                if (free_list[i].second >= bytes && free_list[i].second <= 2 * bytes + (1 << 20) &&
                    (best == free_list.size() || free_list[i].second < free_list[best].second))
                    best = i;
            if (best < free_list.size()) {
                void* p = free_list[best].first;
                *got = free_list[best].second;
                free_list.erase(free_list.begin() + (long)best);
                return p;
            }
        }
        void* p = nullptr;
        if (cudaMallocHost(&p, bytes) != cudaSuccess) { cudaGetLastError(); return nullptr; }
        *got = bytes;
        return p;
    }
    void give(void* p, size_t bytes) {
        if (!p) return;
        std::lock_guard<std::mutex> lk(mu);
        if (free_list.size() >= 8) {                       // keep the 8 largest
            size_t smallest = 0;
            for (size_t i = 1; i < free_list.size(); ++i)
                if (free_list[i].second < free_list[smallest].second) smallest = i;
            if (free_list[smallest].second >= bytes) { cudaFreeHost(p); return; }
            cudaFreeHost(free_list[smallest].first);
            free_list.erase(free_list.begin() + (long)smallest);
        }
        free_list.emplace_back(p, bytes);
    }
    void* lease(size_t bytes) {
        size_t got = 0;
        void* p = take(bytes, &got);
        if (!p) return nullptr;
        std::lock_guard<std::mutex> lk(mu);
        leased.emplace_back(p, got);
        return p;
    }
    void release(void* p) {
        size_t bytes = 0;
        {
            std::lock_guard<std::mutex> lk(mu);
            for (size_t i = 0; i < leased.size(); ++i)
                if (leased[i].first == p) { bytes = leased[i].second; leased.erase(leased.begin() + (long)i); break; }
        }
        if (bytes) give(p, bytes);
    }
};
PinnedPool g_pinned_pool;

// Fill h->stats from the last run's stream-ordered counter copy and stage events (blocks until that run is done).
int resolve_stats(b200gate_handle* h) {
    if (!h->stats_pending) return B200GATE_OK;
    h->stats_pending = false;
    cudaError_t e = cudaEventSynchronize(h->ev_done);
    if (e != cudaSuccess) return fail(h, B200GATE_ERR_CUDA, "CUDA error: %s", cudaGetErrorString(e));
    const Counters cnt = *h->h_cnt;
    float ms = 0.f;
    cudaEventElapsedTime(&ms, h->ev0, h->ev1);
    h->stats.bins_rechecked_fp64 = (int64_t)cnt.rechecked;
    h->stats.bins_unresolved = (int64_t)cnt.unresolved;
    h->stats.rowfloor_flags = (int64_t)cnt.floor_flags;
    h->stats.rowfloor_ambiguous = (int64_t)cnt.floor_ambiguous;
    h->stats.last_run_ms = ms;
    for (size_t b = 0; b < h->pend_batches; ++b) {
        float t1 = 0.f, t2 = 0.f, t3 = 0.f;
        cudaEventElapsedTime(&t1, h->stage_ev[4 * b + 0], h->stage_ev[4 * b + 1]);
        cudaEventElapsedTime(&t2, h->stage_ev[4 * b + 1], h->stage_ev[4 * b + 2]);
        cudaEventElapsedTime(&t3, h->stage_ev[4 * b + 2], h->stage_ev[4 * b + 3]);
        h->stats.k1_ms += t1;
        h->stats.smooth_ms += t2;
        h->stats.k2_ms += t3;
    }
    return B200GATE_OK;
}

}  // namespace

// =============================================================================================
extern "C" {

int b200gate_create(const b200gate_params* p, b200gate_handle** out) {
    if (!p || !out) return fail(nullptr, B200GATE_ERR_ARG, "null argument");
    *out = nullptr;
    if (p->abi_version != B200GATE_ABI_VERSION)
        return fail(nullptr, B200GATE_ERR_ARG, "ABI version %d, library is %d", p->abi_version, B200GATE_ABI_VERSION);
    if (p->surface != B200GATE_SURFACE_NUMPY && p->surface != B200GATE_SURFACE_TORCH &&
        p->surface != B200GATE_SURFACE_TORCH_CHUNKED)
        return fail(nullptr, B200GATE_ERR_ARG, "unknown surface %d", p->surface);
    const bool geo1k = p->n_fft == kN && p->win_length == kN && p->hop_length == kN / 4;
    const bool geo2k = p->n_fft == kN2 && p->win_length == kN2 && p->hop_length == kN2 / 4 &&
                       p->surface == B200GATE_SURFACE_NUMPY && !p->stationary;
    // everything else the reference accepts on the numpy surface runs on the general-geometry family
    // (path_flags bit 2 forces it for the tuned geometries too: the float64 cross-check of the fast kernels)
    // ... and so does a smoothing filter beyond what the tuned integer kernels hold (16-bit mask numerators, 64 taps a side)
    const bool big_filter = p->n_grad_freq > 64 || p->n_grad_time > 64 ||
                            (long long)(p->n_grad_freq + 1) * (p->n_grad_freq + 1) * (p->n_grad_time + 1) * (p->n_grad_time + 1) > 65535;
    // the chunked torch surface always runs it: the reference feeds TorchGate float64 chunks (base.py:140)
    const bool want_generic = (!geo1k && !geo2k) || (p->path_flags & 4) || big_filter ||
                              p->surface == B200GATE_SURFACE_TORCH_CHUNKED;
    int logN = 0;
    while ((1 << logN) < p->n_fft) ++logN;
    if (want_generic) {
        const bool pow2 = (1 << logN) == p->n_fft;
        const bool size_ok = p->n_fft >= 8 && p->n_fft <= (pow2 ? 8192 : 4096);
        if (!size_ok || p->win_length < 1 || p->win_length > p->n_fft || p->hop_length < 1 || p->hop_length > p->win_length)
            return fail(nullptr, B200GATE_ERR_ARG,
                        "unsupported STFT geometry n_fft=%d win_length=%d hop_length=%d (%s gate, %s surface): n_fft must "
                        "be in [8, 8192] if a power of two, else in [8, 4096], with 1 <= hop_length <= win_length <= n_fft",
                        p->n_fft, p->win_length, p->hop_length, p->stationary ? "stationary" : "non-stationary",
                        p->surface == B200GATE_SURFACE_NUMPY ? "numpy" : "torch");
    }
    if (p->n_grad_freq < 0 || p->n_grad_time < 0 || p->n_grad_freq > 65535 || p->n_grad_time > 65535)
        return fail(nullptr, B200GATE_ERR_ARG, "smoothing extents out of range (%d, %d)", p->n_grad_freq, p->n_grad_time);
    if (p->padding < 0) return fail(nullptr, B200GATE_ERR_ARG, "padding must be >= 0");
    // TorchGate asserts 0 <= prop_decrease <= 1 (torchgate.py:52); reduce_noise() takes any value (stationary.py:108)
    if (!std::isfinite(p->prop_decrease) ||
        (p->surface != B200GATE_SURFACE_NUMPY && !(p->prop_decrease >= 0.0 && p->prop_decrease <= 1.0)))
        return fail(nullptr, B200GATE_ERR_ARG, "prop_decrease must be finite (and in [0, 1] on the torch surface)");
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
        return fail(nullptr, B200GATE_ERR_CUDA, "no CUDA device (%s); this library has no CPU fallback",
                    e == cudaSuccess ? "device count 0" : cudaGetErrorString(e));
    b200gate_handle* h = new b200gate_handle();
    h->p = *p;
    int dev = 0;
    cudaGetDevice(&dev);
    h->device = dev;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, dev) == cudaSuccess) h->num_sm = prop.multiProcessorCount;
    if (p->reserve_sms > 0 && p->reserve_sms < h->num_sm) h->num_sm -= p->reserve_sms;   // leave room for NCCL
    h->generic = want_generic;
    h->g_logN = logN;
    if (want_generic && (1 << logN) != p->n_fft) {              // Bluestein: M = 2^k >= 2 n_fft - 1
        while ((1 << h->g_logM) < 2 * p->n_fft - 1) ++h->g_logM;
        h->g_M = 1 << h->g_logM;
    }
    h->F = want_generic ? p->n_fft / 2 + 1 : (p->n_fft == kN2 ? kF2 : kF);
    int rc = want_generic ? build_generic_tables(h) : build_static_tables(h);
    if (rc == B200GATE_OK) {
        e = cudaMalloc((void**)&h->d_cnt, sizeof(Counters));
        if (e == cudaSuccess) e = cudaMalloc((void**)&h->d_need_rowmax, sizeof(unsigned));
        if (e == cudaSuccess) e = cudaMallocHost((void**)&h->h_cnt, sizeof(Counters));
        if (e == cudaSuccess) e = cudaEventCreate(&h->ev0);
        if (e == cudaSuccess) e = cudaEventCreate(&h->ev1);
        if (e == cudaSuccess) e = cudaEventCreate(&h->ev_done);
        if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&h->s_h2d, cudaStreamNonBlocking);
        if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&h->s_d2h, cudaStreamNonBlocking);
        if (e != cudaSuccess) rc = fail(h, B200GATE_ERR_CUDA, "handle resources: %s", cudaGetErrorString(e));
    }
    if (rc == B200GATE_OK) {
#ifndef B200_CUSIM_BUILD
        for (int dt = 0; dt < 3; ++dt)
            B200_WITH_DTYPE(dt, {
                cudaFuncSetAttribute(k1_analyze<8, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, k1_smem_floats() * 4);
                cudaFuncSetAttribute(k1_analyze<8, T, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, k1_smem_floats() * 4);
                cudaFuncSetAttribute(k2_synthesize<8, false, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, k2_smem_floats(256) * 4);
                cudaFuncSetAttribute(k2_synthesize<8, true, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, k2_smem_floats(256) * 4);
                cudaFuncSetAttribute(k1n_magnitude<8, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, k1n_smem_floats() * 4);
                cudaFuncSetAttribute(k1d_analyze<8, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, k1d_smem_bytes());
                cudaFuncSetAttribute(k2d_synthesize<8, false, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, k2d_smem_bytes());
                cudaFuncSetAttribute(k2d_synthesize<8, true, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, k2d_smem_bytes());
                cudaFuncSetAttribute(k2c_synthesize<8, kMaskU16, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, k2c_smem_bytes<kMaskU16>());
                cudaFuncSetAttribute(k2c_synthesize<8, kMaskU16Blend, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, k2c_smem_bytes<kMaskU16Blend>());
                cudaFuncSetAttribute(k2c_synthesize<8, kMaskF32, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, k2c_smem_bytes<kMaskF32>());
                cudaFuncSetAttribute(k2c_synthesize<8, kMaskBits, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, k2c_smem_bytes<kMaskBits>());
                cudaFuncSetAttribute(k2c_synthesize<8, kMaskBitsBlend, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, k2c_smem_bytes<kMaskBitsBlend>());
            });
        cudaFuncSetAttribute(k_smooth_f, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
        cudaFuncSetAttribute(k_smooth_stream<>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
        for (int nfb = 1; nfb <= 12; ++nfb) smooth_box_dispatch(SmoothFArgs{}, nfb, dim3(1), 0, nullptr, true);
        // b200gate_run_rows: the ROWS instantiations of the default kernel selection
        for (int dt = 0; dt < 3; ++dt)
            B200_WITH_DTYPE(dt, {
                cudaFuncSetAttribute(k1_analyze<8, T, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, k1_smem_floats() * 4);
                cudaFuncSetAttribute(k1_analyze<8, T, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, k1_smem_floats() * 4);
                cudaFuncSetAttribute(k1_analyze<8, T, false, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, k1_smem_floats() * 4);
                cudaFuncSetAttribute(k1_analyze<8, T, true, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, k1_smem_floats() * 4);
                cudaFuncSetAttribute(k1n_magnitude<8, T, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, k1n_smem_floats() * 4);
                cudaFuncSetAttribute(k2c_synthesize<8, kMaskF32, T, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, k2c_smem_bytes<kMaskF32>());
                cudaFuncSetAttribute(k2c_synthesize<8, kMaskBits, T, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, k2c_smem_bytes<kMaskBits>());
                cudaFuncSetAttribute(k2c_synthesize<8, kMaskBitsBlend, T, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, k2c_smem_bytes<kMaskBitsBlend>());
            });
        cudaFuncSetAttribute(k_smooth_stream<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
        for (int nfb = 1; nfb <= 12; ++nfb) smooth_box_dispatch<true>(SmoothFArgs{}, nfb, dim3(1), 0, nullptr, true);
        // (torch surface, stationary extents beyond the in-synthesis smoothing: numerators from k_smooth_generic)
        cudaFuncSetAttribute(k_smooth_generic<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024);
        // b200gate_tstream_*: the STREAM instantiations
        cudaFuncSetAttribute(k1n_magnitude<8, float, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, k1n_smem_floats() * 4);
        cudaFuncSetAttribute(k2c_synthesize<8, kMaskF32, float, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             k2c_smem_bytes<kMaskF32>());
        cudaFuncSetAttribute(k_smooth_stream<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
        for (int nfb = 1; nfb <= 12; ++nfb) smooth_box_dispatch<false, true>(SmoothFArgs{}, nfb, dim3(1), 0, nullptr, true);
        // b200gate_tstream_push_rows / _end_rows: the SESS instantiations
        cudaFuncSetAttribute(k1n_magnitude<8, float, false, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             k1n_smem_floats() * 4);
        cudaFuncSetAttribute(k2c_synthesize<8, kMaskF32, float, false, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             k2c_smem_bytes<kMaskF32>());
        cudaFuncSetAttribute(k_smooth_stream<false, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
        for (int nfb = 1; nfb <= 12; ++nfb) smooth_box_dispatch<false, true, true>(SmoothFArgs{}, nfb, dim3(1), 0, nullptr, true);
        cudaFuncSetAttribute(k2c_synthesize<8, kMaskU16, float, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, k2c_smem_bytes<kMaskU16>());
        cudaFuncSetAttribute(k2c_synthesize<8, kMaskU16Blend, float, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, k2c_smem_bytes<kMaskU16Blend>());
        cudaFuncSetAttribute(k1n_magnitude_2k, cudaFuncAttributeMaxDynamicSharedMemorySize, k1n2_smem_floats() * 4);
        cudaFuncSetAttribute(k2_synthesize_2k<>, cudaFuncAttributeMaxDynamicSharedMemorySize, k22_smem_floats() * 4);
        cudaFuncSetAttribute(k2_synthesize_2k<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, k22_smem_floats() * 4);
        cudaFuncSetAttribute(k2c_synthesize_2k, cudaFuncAttributeMaxDynamicSharedMemorySize, k2c2_smem_bytes());
        cudaFuncSetAttribute(k_smooth_generic<>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024);
        for (int dt = 0; dt < 3; ++dt)
            B200_WITH_DTYPE(dt, { cudaFuncSetAttribute(gk_stft<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, 8192 * 16); });
        cudaFuncSetAttribute(gk_istft, cudaFuncAttributeMaxDynamicSharedMemorySize, 8192 * 16);
        // the adjoint (b200gate_adjoint): float32 / float64 gradients
        cudaFuncSetAttribute(k2_synthesize<8, false, float, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, k2_smem_floats(256) * 4);
        cudaFuncSetAttribute(k2_synthesize<8, true, float, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, k2_smem_floats(256) * 4);
        cudaFuncSetAttribute(k2_synthesize<8, false, double, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, k2_smem_floats(256) * 4);
        cudaFuncSetAttribute(k2_synthesize<8, true, double, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, k2_smem_floats(256) * 4);
        cudaFuncSetAttribute(gk_stft<float, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 8192 * 16);
        cudaFuncSetAttribute(gk_stft<double, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 8192 * 16);
#endif
    }
    if (rc != B200GATE_OK) {
        g_create_error = h->err;
        b200gate_destroy(h);
        return rc;
    }
    *out = h;
    return B200GATE_OK;
}

void b200gate_destroy(b200gate_handle* h) {
    if (!h) return;
    int cur_dev = 0;
    cudaGetDevice(&cur_dev);
    if (cur_dev != h->device) cudaSetDevice(h->device);
    cudaDeviceSynchronize();                                 // nothing of this handle is in flight when its buffers change hands
    g_device_pool.give(h->d_ws_buf, h->ws_bytes, h->device);
    g_device_pool.give(h->d_in, h->in_bytes, h->device);
    g_device_pool.give(h->d_out, h->out_bytes, h->device);
    g_device_pool.give(h->d_raw, h->raw_bytes, h->device);
    g_device_pool.give(h->d_swin, h->swin_bytes, h->device);
    g_device_pool.give(h->d_sout, h->sout_bytes, h->device);
    void* ptrs[] = {h->d_wa, h->d_ws, h->d_invn, h->d_thr4, h->d_gco, h->d_floor4, h->d_ef, h->d_tw, h->d_thr2_64,
                    h->d_wa64, h->d_cs64, h->d_tthr, h->d_wa2, h->d_ws2, h->d_w2k, h->d_invn2, h->d_cnt, h->d_dbg_spec,
                    h->d_dbg_mask, h->d_dbg_bits, h->d_gwa, h->d_gws, h->d_gw2, h->d_gthr, h->d_gcs, h->d_gtthr, h->d_gchirp, h->d_gbbr};
    for (void* p : ptrs)
        if (p) cudaFree(p);
    if (h->ev0) cudaEventDestroy(h->ev0);
    if (h->ev1) cudaEventDestroy(h->ev1);
    if (h->ev_done) cudaEventDestroy(h->ev_done);
    for (cudaEvent_t e : h->group_ev) cudaEventDestroy(e);
    if (h->h_cnt) cudaFreeHost(h->h_cnt);
    for (int i = 0; i < 2; ++i) { g_pinned_pool.give(h->hp_in[i], h->hp_in_bytes[i]); g_pinned_pool.give(h->hp_out[i], h->hp_out_bytes[i]); }
    if (h->d_need_rowmax) cudaFree(h->d_need_rowmax);
    g_pinned_pool.give(h->hp_units, h->hp_units_bytes);
    g_pinned_pool.give(h->hp_sess, h->hp_sess_bytes);
    for (cudaEvent_t e : h->ev_sess) cudaEventDestroy(e);
    if (h->d_units) cudaFree(h->d_units);
    if (h->d_rtab) cudaFree(h->d_rtab);
    if (h->d_ts) cudaFree(h->d_ts);
    if (h->ev_units) cudaEventDestroy(h->ev_units);
    for (cudaEvent_t e : h->stage_ev) cudaEventDestroy(e);
    for (cudaEvent_t e : h->pipe_ev) cudaEventDestroy(e);
    if (h->s_h2d) cudaStreamDestroy(h->s_h2d);
    if (h->s_d2h) cudaStreamDestroy(h->s_d2h);
    for (int i = 0; i < 2; ++i) {
        g_device_pool.give(h->d_slab_in[i], h->slab_in_bytes[i], h->device);
        g_device_pool.give(h->d_slab_out[i], h->slab_out_bytes[i], h->device);
    }
    if (cur_dev != h->device) cudaSetDevice(cur_dev);
    delete h;
}

const char* b200gate_last_error(const b200gate_handle* h) { return h ? h->err.c_str() : g_create_error.c_str(); }

int b200gate_set_noise_threshold(b200gate_handle* h, const double* thresh_db, int32_t n_bins) {
    if (!h || !thresh_db) return B200GATE_ERR_ARG;
    const int F = h->generic ? h->F : kF;
    if (n_bins != F) return fail(h, B200GATE_ERR_ARG, "expected %d bins, got %d", F, n_bins);
    h->thr.assign(thresh_db, thresh_db + F);
    h->mean.assign(F, NAN);
    h->sd.assign(F, NAN);
    if (h->generic) {
        int rc = upload(h, &h->d_gthr, h->thr);
        if (rc == B200GATE_OK) h->have_thresh = true;
        return rc;
    }
    return build_threshold_tables(h);
}

int b200gate_set_noise_threshold_rows(b200gate_handle* h, const double* thresh_db, int64_t n_recordings, int32_t n_bins) {
    if (!h || !thresh_db || n_recordings <= 0) return fail(h, B200GATE_ERR_ARG, "bad argument");
    const b200gate_params& p = h->p;
    if (!p.stationary || p.surface != B200GATE_SURFACE_NUMPY || h->generic || p.n_fft != kN)
        return fail(h, B200GATE_ERR_ARG, "per-recording thresholds are for the stationary numpy-surface gate at n_fft 1024");
    if (n_bins != kF) return fail(h, B200GATE_ERR_ARG, "expected %d bins, got %d", kF, n_bins);
    if (n_recordings > 0x7fffffffLL / kFPad) return fail(h, B200GATE_ERR_ARG, "too many recordings");
    const size_t R = (size_t)n_recordings;
    // one host image of the tables (the layout of rec_tables()), one upload
    const size_t fl = 3 * R * kFPad;                       // (3 kFPad floats are a whole number of doubles)
    std::vector<double> img(fl / 2 + R * kF);
    float* f = (float*)img.data();
    double* t2 = img.data() + fl / 2;
    for (size_t r = 0; r < R; ++r) {
        float *thr4 = f + r * kFPad, *gco = f + (R + r) * kFPad, *floor4 = f + (2 * R + r) * kFPad;
        std::fill(thr4, thr4 + kFPad, INFINITY);
        std::fill(gco, gco + kFPad, 0.f);
        std::fill(floor4, floor4 + kFPad, INFINITY);
        const double mfa = threshold_rows(p, thresh_db + r * kF, thr4, gco, floor4, t2 + r * kF);
        floor4[kFPad - 1] = (float)(4.0 * mfa * mfa);      // the recording's need_rowmax guard (k1_analyze<.., PERREC>)
    }
    const size_t bytes = img.size() * sizeof(double);
    if (h->rtab_bytes < bytes) {
        if (h->d_rtab) cudaFree(h->d_rtab);
        h->d_rtab = nullptr;
        h->rtab_bytes = 0;
        h->n_rec = 0;
        CK(h, cudaMalloc(&h->d_rtab, bytes));
        h->rtab_bytes = bytes;
    }
    CK(h, cudaMemcpy(h->d_rtab, img.data(), bytes, cudaMemcpyHostToDevice));
    h->n_rec = (int)R;
    h->have_thresh = false;                                // (b200gate_run, get_noise_threshold, streams: ERR_STATE)
    return B200GATE_OK;
}

int b200gate_get_noise_threshold(const b200gate_handle* h, double* thresh_db, int32_t n_bins) {
    if (!h || !thresh_db || n_bins != (h->generic ? h->F : kF) || !h->have_thresh) return B200GATE_ERR_STATE;
    memcpy(thresh_db, h->thr.data(), (size_t)n_bins * sizeof(double));
    return B200GATE_OK;
}

int b200gate_get_noise_mean_std(const b200gate_handle* h, double* mean_db, double* std_db, int32_t n_bins) {
    if (!h || n_bins != (h->generic ? h->F : kF) || !h->have_thresh) return B200GATE_ERR_STATE;
    if (mean_db) memcpy(mean_db, h->mean.data(), (size_t)n_bins * sizeof(double));
    if (std_db) memcpy(std_db, h->sd.data(), (size_t)n_bins * sizeof(double));
    return B200GATE_OK;
}

int b200gate_set_window(b200gate_handle* h, const float* window, int32_t win_length) {
    if (!h || !window) return B200GATE_ERR_ARG;
    if (h->generic) {
        if (win_length != h->p.win_length) return fail(h, B200GATE_ERR_ARG, "window length %d != win_length %d", win_length, h->p.win_length);
        h->user_window.assign(window, window + win_length);
        return build_generic_tables(h);
    }
    if (win_length != h->p.n_fft) return fail(h, B200GATE_ERR_ARG, "window length %d != n_fft %d", win_length, h->p.n_fft);
    h->user_window.assign(window, window + win_length);
    return build_static_tables(h);
}

}  // extern "C"

namespace {
// run `stmt` with the constant D bound to the format code `dt` (any code cv_size knows)
#define B200_WITH_FORMAT(dt, ...)                                                                          \
    switch (dt) {                                                                                          \
        case B200GATE_F32: { constexpr int D = B200GATE_F32; __VA_ARGS__; } break;                          \
        case B200GATE_I16: { constexpr int D = B200GATE_I16; __VA_ARGS__; } break;                          \
        case B200GATE_F64: { constexpr int D = B200GATE_F64; __VA_ARGS__; } break;                          \
        case B200GATE_BOOL: { constexpr int D = B200GATE_BOOL; __VA_ARGS__; } break;                        \
        case B200GATE_I8: { constexpr int D = B200GATE_I8; __VA_ARGS__; } break;                            \
        case B200GATE_U8: { constexpr int D = B200GATE_U8; __VA_ARGS__; } break;                            \
        case B200GATE_U16: { constexpr int D = B200GATE_U16; __VA_ARGS__; } break;                          \
        case B200GATE_I32: { constexpr int D = B200GATE_I32; __VA_ARGS__; } break;                          \
        case B200GATE_U32: { constexpr int D = B200GATE_U32; __VA_ARGS__; } break;                          \
        case B200GATE_I64: { constexpr int D = B200GATE_I64; __VA_ARGS__; } break;                          \
        case B200GATE_U64: { constexpr int D = B200GATE_U64; __VA_ARGS__; } break;                          \
        default: { constexpr int D = B200GATE_F16; __VA_ARGS__; } break;                                   \
    }

// elementwise, bandwidth-bound: enough CTAs to fill the device, each striding over a row's columns
dim3 convert_grid(long long C, long long N) {
    const int gy = (int)std::min<long long>(C, 1024);
    return dim3(grid_1d(N, 256, std::max(1, 4096 / gy)), gy);
}
}  // namespace

extern "C" {

int b200gate_convert(int op, const void* src, int src_dtype, int64_t src_stride, void* dst, int dst_dtype,
                     int64_t dst_stride, int64_t C, int64_t N, void* stream) {
    if (((!src || !dst) && C > 0 && N > 0) || C < 0 || N < 0 || cv_size(src_dtype) == 0 || cv_size(dst_dtype) == 0 ||
        (C > 1 && src_stride < N))
        return fail(nullptr, B200GATE_ERR_ARG, "b200gate_convert: bad argument");
    cudaStream_t st = (cudaStream_t)stream;
    if (op == B200GATE_CONVERT_CAST) {
        if (src_dtype != B200GATE_F64 && dst_dtype != B200GATE_F64)
            return fail(nullptr, B200GATE_ERR_ARG, "b200gate_convert: a cast goes to or from float64");
        if (C > 1 && dst_stride < N) return fail(nullptr, B200GATE_ERR_ARG, "b200gate_convert: dst_stride < N");
        if (C == 0 || N == 0) return B200GATE_OK;
        const dim3 grid = convert_grid(C, N);
        if (dst_dtype == B200GATE_F64) {
            B200_WITH_FORMAT(src_dtype, { auto kern_ = k_convert<D, B200GATE_F64>;
                B200_LAUNCH(kern_, grid, dim3(256), 0, st, src, (long long)src_stride, dst, (long long)dst_stride, (long long)C, (long long)N); });
        } else {
            B200_WITH_FORMAT(dst_dtype, { auto kern_ = k_convert<B200GATE_F64, D>;
                B200_LAUNCH(kern_, grid, dim3(256), 0, st, src, (long long)src_stride, dst, (long long)dst_stride, (long long)C, (long long)N); });
        }
    } else if (op == B200GATE_CONVERT_CHANNEL_MEAN) {
        if (dst_dtype != B200GATE_F64 || C == 0)
            return fail(nullptr, B200GATE_ERR_ARG, "b200gate_convert: the channel mean takes C >= 1 and a float64 dst");
        if (N == 0) return B200GATE_OK;
        B200_WITH_FORMAT(src_dtype, { auto kern_ = k_channel_mean<D>;
            B200_LAUNCH(kern_, dim3(grid_1d(N, 256, 4096)), dim3(256), 0, st, src, (long long)src_stride, (double*)dst, (long long)C, (long long)N); });
    } else {
        return fail(nullptr, B200GATE_ERR_ARG, "b200gate_convert: unknown operation %d", op);
    }
    CK(nullptr, cudaGetLastError());
    return B200GATE_OK;
}

int b200gate_channel_sum(b200gate_handle* h, const void* y, int dtype, int64_t C, int64_t n, int64_t stride,
                         int is_device, void* acc, int init, void* stream) {
    if (!h || !y || !acc || C <= 0 || n <= 0 || dtype_size(dtype) == 0) return fail(h, B200GATE_ERR_ARG, "bad argument");
    return channel_sum_impl(h, y, dtype, C, n, stride, is_device, acc, init, (cudaStream_t)stream);
}

void* b200gate_host_alloc(size_t bytes) {
    if (bytes == 0) return nullptr;
#ifdef B200_CUSIM_BUILD
    return malloc(bytes);
#else
    return g_pinned_pool.lease(bytes);
#endif
}
void b200gate_host_free(void* p) {
    if (!p) return;
#ifdef B200_CUSIM_BUILD
    free(p);
#else
    g_pinned_pool.release(p);
#endif
}

int b200gate_noise_stats_collapsed(b200gate_handle* h, const void* noise_mean, int dtype, int64_t n, int is_device,
                                   void* stream) {
    if (!h || !noise_mean || n <= 0) return fail(h, B200GATE_ERR_ARG, "bad argument");
    if (dtype != B200GATE_F32 && dtype != B200GATE_F64) return fail(h, B200GATE_ERR_ARG, "collapsed noise must be f32 or f64");
    cudaStream_t st = (cudaStream_t)stream;
    const size_t es = dtype_size(dtype);
    Scratch s_src, s_yn;
    CK(h, s_yn.alloc((size_t)n * sizeof(double)));
    double* d_yn = s_yn.as<double>();
    const void* src = noise_mean;
    if (!is_device) {
        CK(h, s_src.alloc((size_t)n * es));
        CK(h, cudaMemcpyAsync(s_src.p, noise_mean, (size_t)n * es, cudaMemcpyHostToDevice, st));
        src = s_src.p;
    }
    if (dtype == B200GATE_F32)
        { auto kern_ = k0_mean_to_f64<float>; B200_LAUNCH(kern_, dim3(grid_1d(n, 256, 4096)), dim3(256), 0, st, (const float*)src, (long long)n, 1LL, d_yn); }
    else
        { auto kern_ = k0_mean_to_f64<double>; B200_LAUNCH(kern_, dim3(grid_1d(n, 256, 4096)), dim3(256), 0, st, (const double*)src, (long long)n, 1LL, d_yn); }
    return noise_stats_from_mean(h, d_yn, n, st);          // synchronises the stream before the scratch is freed
}

int b200gate_noise_stats(b200gate_handle* h, const void* y_noise, int dtype, int64_t C, int64_t N, int64_t stride,
                         int is_device, void* stream) {
    if (!h || !y_noise || C <= 0 || N <= 0 || dtype_size(dtype) == 0) return fail(h, B200GATE_ERR_ARG, "bad argument");
    cudaStream_t st = (cudaStream_t)stream;
    long long n = N;
    if (h->p.clip_noise && h->p.chunk_size > 0 && n > h->p.chunk_size) n = h->p.chunk_size;   // stationary.py:63-64
    const bool f32 = (dtype == B200GATE_F32);
    Scratch s_acc, s_yn;
    CK(h, s_acc.alloc((size_t)n * (f32 ? 4 : 8)));
    CK(h, s_yn.alloc((size_t)n * sizeof(double)));
    void* d_acc = s_acc.p;
    double* d_yn = s_yn.as<double>();
    int rc = channel_sum_impl(h, y_noise, dtype, C, n, stride, is_device, d_acc, 1, st);
    if (rc == B200GATE_OK) {
        if (f32)
            { auto kern_ = k0_mean_to_f64<float>; B200_LAUNCH(kern_, dim3(grid_1d(n, 256, 4096)), dim3(256), 0, st, (const float*)d_acc, n, (long long)C, d_yn); }
        else
            { auto kern_ = k0_mean_to_f64<double>; B200_LAUNCH(kern_, dim3(grid_1d(n, 256, 4096)), dim3(256), 0, st, (const double*)d_acc, n, (long long)C, d_yn); }
        rc = noise_stats_from_mean(h, d_yn, n, st);
    }
    return rc;
}

}  // extern "C"

namespace {
// host clips: channel-order sums of samples [i0, i1) into a, the additions of channel_sum_impl's host path
template <typename Tin, typename Tacc>
void host_channel_sum(const Tin* y, long long C, long long stride, long long i0, long long i1, Tacc* a) {
    for (long long i = i0; i < i1; ++i) a[i] = (Tacc)0;
    for (long long c = 0; c < C; ++c) {
        const Tin* r = y + c * stride;
        for (long long i = i0; i < i1; ++i) a[i] = a[i] + (Tacc)r[i];
    }
}
}  // namespace

extern "C" {

// Thresholds of many clips: one K0Clip table, then per group of clips (under the workspace limit) one launch each of
// k0_clip_mean_rows, k0_stft_db_rows and k0_stats_rows; the thresholds of every clip are read back at the end, once.
int b200gate_noise_stats_rows(b200gate_handle* h, const b200gate_noise_clip* clips, int64_t n_clips, int dtype,
                              int is_device, double* thresh_out, void* stream) {
    if (!h || !clips || n_clips <= 0 || !thresh_out || dtype_size(dtype) == 0) return fail(h, B200GATE_ERR_ARG, "bad argument");
    const b200gate_params& p = h->p;
    if (h->generic || p.n_fft != kN || p.win_length != kN || p.hop_length != kN / 4)
        return fail(h, B200GATE_ERR_ARG, "b200gate_noise_stats_rows needs n_fft = win_length = 1024, hop_length = 256");
    cudaStream_t st = (cudaStream_t)stream;
    const int H = p.hop_length;
    const bool f32 = dtype == B200GATE_F32;
    const size_t as = f32 ? 4 : 8;                             // accumulation dtype of the channel sum
    std::vector<K0Clip> tab((size_t)n_clips);
    long long n_sum = 0;                                       // host clips: samples of all their channel sums
    for (int64_t r = 0; r < n_clips; ++r) {
        const b200gate_noise_clip& c = clips[r];
        if (!c.x || c.C <= 0 || c.n <= 0 || (c.C > 1 && c.stride < c.n))
            return fail(h, B200GATE_ERR_ARG, "clip %lld: null pointer, no samples or channels, or a row stride below n", (long long)r);
        long long n = c.n;
        if (p.clip_noise && p.chunk_size > 0 && n > p.chunk_size) n = p.chunk_size;       // stationary.py:63-64
        if (n < p.win_length)                                  // (scipy would shorten the window: b200gate_noise_stats on
            return fail(h, B200GATE_ERR_ARG, "clip %lld: %lld samples after clipping, fewer than win_length %d "
                        "(b200gate_noise_stats takes such a clip on a handle with win_length = n)", (long long)r, n, p.win_length);
        K0Clip& k = tab[(size_t)r];
        k.x = c.x; k.stride = c.stride; k.c_sum = c.C; k.C = c.C; k.n = n; k.Tn = (int)(n / H) + 1;
        if (!is_device) {                                      // (x is set to the device copy of its sums below)
            k.yn_off = n_sum;
            n_sum += n;
        }
    }
    // host clips: their channel sums are taken by the host workers, the same additions in the same type as
    // k0_channel_sum, and only the sums travel, with the table, in one pinned buffer and one copy
    const size_t tab_bytes = tab.size() * sizeof(K0Clip), sum_off = (tab_bytes + 255) / 256 * 256;
    const size_t up_bytes = sum_off + (is_device ? 0 : (size_t)n_sum * as);
    size_t pinned_bytes = 0;
    void* hp = g_pinned_pool.take(up_bytes, &pinned_bytes);
    if (!hp) return fail(h, B200GATE_ERR_NOMEM, "pinned staging (%zu bytes)", up_bytes);
    struct PinnedBack {
        void* p; size_t b;
        ~PinnedBack() { g_pinned_pool.give(p, b); }            // (after the synchronise below, or on an early return)
    } pinned_back{hp, pinned_bytes};
    Scratch s_up;
    CK(h, s_up.alloc(up_bytes));
    const K0Clip* d_tab = s_up.as<K0Clip>();
    if (!is_device) {
        unsigned char* hsum = (unsigned char*)hp + sum_off;
        const long long blk = 8192;
        std::vector<std::pair<int64_t, long long>> jobs;        // (clip, first sample of a block)
        for (int64_t r = 0; r < n_clips; ++r)
            for (long long i0 = 0; i0 < tab[(size_t)r].n; i0 += blk) jobs.emplace_back(r, i0);
        const int nt = (int)std::max<size_t>(1, std::min<size_t>((size_t)std::min(h->host_threads, 32), jobs.size()));
        std::function<void(int)> work = [&](int id) {
            for (size_t j = (size_t)id; j < jobs.size(); j += (size_t)nt) {
                const K0Clip& k = tab[(size_t)jobs[j].first];
                const long long i0 = jobs[j].second, i1 = std::min(k.n, i0 + blk);
                void* a = hsum + (size_t)k.yn_off * as;
                if (dtype == B200GATE_F32) host_channel_sum((const float*)k.x, k.C, k.stride, i0, i1, (float*)a);
                else if (dtype == B200GATE_I16) host_channel_sum((const short*)k.x, k.C, k.stride, i0, i1, (double*)a);
                else host_channel_sum((const double*)k.x, k.C, k.stride, i0, i1, (double*)a);
            }
        };
        host_workers(0).run(nt, work);
        for (K0Clip& k : tab) {
            k.x = (const char*)s_up.p + sum_off + (size_t)k.yn_off * as;
            k.stride = k.n;
            k.c_sum = 1;
        }
    }
    // groups of clips whose float64 means and dB spectrograms fit the workspace limit (at least one clip each)
    double limit = p.workspace_limit_bytes;
    if (!(limit > 0)) {
        limit = 24.0 * 1024 * 1024 * 1024;
        size_t free_b = 0, total_b = 0;
        if (cudaMemGetInfo(&free_b, &total_b) == cudaSuccess) limit = std::min(limit, 0.7 * (double)free_b);
    }
    std::vector<int64_t> g_start{0};
    long long yn_max = 0, t_max = 0;
    {
        long long yn = 0, t = 0;
        for (int64_t r = 0; r < n_clips; ++r) {
            K0Clip& k = tab[(size_t)r];
            const double more = 8.0 * ((double)(yn + k.n) + (double)(t + k.Tn) * kF);
            if (r > g_start.back() && (more > limit || r - g_start.back() >= 65535 || t + k.Tn > 0x7fffffffLL)) {
                g_start.push_back(r);
                yn = t = 0;
            }
            k.yn_off = yn;                                     // (host clips' sums were placed above: x holds them)
            k.t_off = t;
            yn += k.n;
            t += k.Tn;
            yn_max = std::max(yn_max, yn);
            t_max = std::max(t_max, t);
        }
        g_start.push_back(n_clips);
    }
    Scratch s_yn, s_db, s_res;
    CK(h, s_yn.alloc((size_t)yn_max * sizeof(double)));
    CK(h, s_db.alloc((size_t)t_max * kF * sizeof(double)));
    CK(h, s_res.alloc((size_t)n_clips * 3 * kF * sizeof(double)));
    memcpy(hp, tab.data(), tab_bytes);
    CK(h, cudaMemcpyAsync(s_up.p, hp, up_bytes, cudaMemcpyHostToDevice, st));
    double *d_yn = s_yn.as<double>(), *d_db = s_db.as<double>(), *d_res = s_res.as<double>();
    for (size_t gi = 0; gi + 1 < g_start.size(); ++gi) {
        const int64_t c0 = g_start[gi], nc = g_start[gi + 1] - c0;
        long long n_hi = 0, frames = 0;
        for (int64_t r = c0; r < c0 + nc; ++r) {
            n_hi = std::max(n_hi, tab[(size_t)r].n);
            frames += tab[(size_t)r].Tn;
        }
        const dim3 gm(grid_1d(n_hi, 256, std::max(1, 4096 / (int)nc)), (unsigned)nc);
        if (f32) {
            auto kern_ = k0_clip_mean_rows<float, float>;
            B200_LAUNCH(kern_, gm, dim3(256), 0, st, d_tab + c0, d_yn);
        } else if (dtype == B200GATE_I16 && is_device) {
            auto kern_ = k0_clip_mean_rows<short, double>;
            B200_LAUNCH(kern_, gm, dim3(256), 0, st, d_tab + c0, d_yn);
        } else {
            auto kern_ = k0_clip_mean_rows<double, double>;
            B200_LAUNCH(kern_, gm, dim3(256), 0, st, d_tab + c0, d_yn);
        }
        K0Args a{};
        a.yn = d_yn; a.H = H; a.wa64 = h->d_wa64; a.cs64 = h->d_cs64; a.eps = kEps64; a.db = d_db;
        B200_LAUNCH(k0_stft_db_rows, dim3((unsigned)frames), dim3(256), kN * sizeof(double2), st, a, d_tab + c0, (int)nc);
        B200_LAUNCH(k0_stats_rows, dim3(kF, (unsigned)nc), dim3(256), 0, st, d_db, d_tab + c0, p.top_db, p.std_ddof,
                    p.n_std_thresh, d_res + (size_t)c0 * 3 * kF);
        CK(h, cudaGetLastError());
    }
    // the thresholds: row 2 of every clip's [3][F] result
    CK(h, cudaMemcpy2DAsync(thresh_out, kF * sizeof(double), d_res + 2 * kF, 3 * kF * sizeof(double), kF * sizeof(double),
                            (size_t)n_clips, cudaMemcpyDeviceToHost, st));
    CK(h, cudaStreamSynchronize(st));
    return B200GATE_OK;
}

int b200gate_debug_select_unit(b200gate_handle* h, int64_t chunk, int64_t channel) {
    if (!h) return B200GATE_ERR_ARG;
    h->dbg_chunk = chunk;
    h->dbg_channel = channel;
    return B200GATE_OK;
}

int b200gate_debug_dims(const b200gate_handle* h, int64_t* T, int32_t* F, int32_t* words) {
    if (!h) return B200GATE_ERR_ARG;
    if (T) *T = h->dbg_T;
    if (F) *F = h->generic ? h->F : (h->p.n_fft == kN2 ? kF2 : kF);
    if (words) *words = h->generic ? (h->F + 31) / 32 : (h->p.n_fft == kN2 ? kFW2 : kFW);
    return B200GATE_OK;
}

int b200gate_debug_read_bits(b200gate_handle* h, uint32_t* bits) {
    if (!h || !bits || !h->d_dbg_bits || h->dbg_T <= 0) return B200GATE_ERR_STATE;
    if (!h->generic && h->p.n_fft == kN2) { memset(bits, 0, (size_t)h->dbg_T * kFW2 * 4); return B200GATE_OK; }   // no binary mask in this family
    CK(h, cudaDeviceSynchronize());
    CK(h, cudaMemcpy(bits, h->d_dbg_bits, (size_t)h->dbg_T * (h->generic ? (h->F + 31) / 32 : kFW) * 4, cudaMemcpyDeviceToHost));
    return B200GATE_OK;
}
int b200gate_debug_read_mask(b200gate_handle* h, float* mask) {
    if (!h || !mask || !h->d_dbg_mask || h->dbg_T <= 0) return B200GATE_ERR_STATE;
    CK(h, cudaDeviceSynchronize());
    CK(h, cudaMemcpy(mask, h->d_dbg_mask, (size_t)h->dbg_T * (h->generic ? h->F : (h->p.n_fft == kN2 ? kF2 : kF)) * 4, cudaMemcpyDeviceToHost));
    return B200GATE_OK;
}
int b200gate_debug_read_spec(b200gate_handle* h, float* spec) {
    if (!h || !spec || !h->d_dbg_spec || h->dbg_T <= 0) return B200GATE_ERR_STATE;
    CK(h, cudaDeviceSynchronize());
    CK(h, cudaMemcpy(spec, h->d_dbg_spec, (size_t)h->dbg_T * (h->generic ? h->F : (h->p.n_fft == kN2 ? kF2 : kF)) * 8, cudaMemcpyDeviceToHost));
    return B200GATE_OK;
}

int b200gate_set_range(b200gate_handle* h, int32_t mode, int64_t a, int64_t b) {
    if (!h) return B200GATE_ERR_ARG;
    if (mode < 0 || mode > 2 || (mode == 1 && (a < 0 || b < a)) || (mode == 2 && a <= 0))
        return fail(h, B200GATE_ERR_ARG, "bad range (mode %d, %lld, %lld)", mode, (long long)a, (long long)b);
    h->range_mode = mode; h->range_a = a; h->range_b = b;
    return B200GATE_OK;
}

int b200gate_get_stats(const b200gate_handle* h, b200gate_stats* out) {
    if (!h || !out) return B200GATE_ERR_ARG;
    const int rc = resolve_stats(const_cast<b200gate_handle*>(h));
    if (rc) return rc;
    *out = h->stats;
    return B200GATE_OK;
}

int b200gate_torch_set_noise(b200gate_handle* h, const void* xn, int dtype, int64_t Bn, int64_t Ln, int64_t stride,
                             int is_device, void* stream) {
    if (!h) return B200GATE_ERR_ARG;
    if (h->p.surface == B200GATE_SURFACE_NUMPY) return fail(h, B200GATE_ERR_STATE, "torch surfaces only");
    if (!xn) { h->tthr_units = 0; return B200GATE_OK; }
    const bool f64 = dtype == B200GATE_F64 && h->generic;            // float64 noise clips: general family only
    if (Bn <= 0 || Ln <= 0 || (dtype != B200GATE_F32 && !f64))
        return fail(h, B200GATE_ERR_ARG, "xn must be float32 [Bn][Ln] (float64 on the general-geometry family)");
    cudaStream_t st = (cudaStream_t)stream;
    const size_t xes = f64 ? 8 : 4;
    const float* x = (const float*)xn;
    Scratch s_tmp;
    long long xs = stride;
    if (!is_device) {
        CK(h, s_tmp.alloc((size_t)Bn * Ln * xes));
        CK(h, cudaMemcpy2DAsync(s_tmp.p, (size_t)Ln * xes, xn, (size_t)stride * xes, (size_t)Ln * xes, (size_t)Bn, cudaMemcpyHostToDevice, st));
        x = s_tmp.as<float>(); xs = Ln;
    }
    Geom g{};
    g.H = h->p.hop_length; g.C = (int)Bn; g.n_total = Ln; g.step = Ln; g.n_chunks = 1; g.pad = 0; g.Lp = Ln;
    g.T = (int)(Ln / g.H) + 1; g.in_stride = xs; g.out_stride = xs; g.u0 = 0; g.n_units = (int)Bn;
    if (h->generic) {                                  // general family: float64 statistics of xn's own frames
        const int F = h->F, N = h->p.n_fft;
        if (Bn > 65535) return fail(h, B200GATE_ERR_ARG, "xn has too many rows");
        Scratch s_gX, s_gD;
        CK(h, s_gX.alloc((size_t)Bn * g.T * F * sizeof(double2)));
        CK(h, s_gD.alloc((size_t)Bn * g.T * F * sizeof(double)));
        double2* gX = s_gX.as<double2>();
        double* gD = s_gD.as<double>();
        if (h->d_gtthr) cudaFree(h->d_gtthr);
        h->d_gtthr = nullptr;
        CK(h, cudaMalloc((void**)&h->d_gtthr, (size_t)Bn * F * sizeof(double)));
        if (f64) {
            GStftArgs<double> sa{};
            sa.gg = generic_geom(h, g); sa.tb = generic_tables(h); sa.x = (const double*)(const void*)x; sa.X = gX;
            auto kern_ = gk_stft<double>;
            B200_LAUNCH(kern_, dim3((unsigned)g.T, (unsigned)Bn), dim3(generic_threads(generic_fft_len(h))), (size_t)generic_fft_len(h) * sizeof(double2), st, sa);
        } else {
            GStftArgs<float> sa{};
            sa.gg = generic_geom(h, g); sa.tb = generic_tables(h); sa.x = x; sa.X = gX;
            auto kern_ = gk_stft<float>;
            B200_LAUNCH(kern_, dim3((unsigned)g.T, (unsigned)Bn), dim3(generic_threads(generic_fft_len(h))), (size_t)generic_fft_len(h) * sizeof(double2), st, sa);
        }
        GTStatArgs ta{};
        ta.n_units = (int)Bn; ta.T = g.T; ta.F = F; ta.ddof = h->p.std_ddof; ta.eps = kEps64; ta.top_db = h->p.top_db;
        ta.n_std = h->p.n_std_thresh; ta.X = gX; ta.scratch = gD; ta.thr = h->d_gtthr;
        B200_LAUNCH(gk_tstats, dim3((unsigned)(((long long)Bn * F + 127) / 128)), dim3(128), 0, st, ta);
        CK(h, cudaGetLastError());
        CK(h, cudaStreamSynchronize(st));
        h->tthr_units = (int)Bn;
        return B200GATE_OK;
    }
    Scratch s_mag, s_rowmax;
    CK(h, s_mag.alloc((size_t)Bn * g.T * kFPad * 4));
    CK(h, s_rowmax.alloc((size_t)Bn * kFPad * 4));
    float *mag = s_mag.as<float>(), *rowmax = s_rowmax.as<float>();
    if (h->d_tthr) cudaFree(h->d_tthr);
    h->d_tthr = nullptr;
    CK(h, cudaMalloc((void**)&h->d_tthr, (size_t)Bn * kFPad * 4));
    DebugTap dbg{}; dbg.ul = -1;
    launch_k1n(g, device_tables(h), x, B200GATE_F32, mag, dbg, h->num_sm * 3, st);
    TStatArgs ta{};
    ta.n_units = (int)Bn; ta.T = g.T; ta.in_scale = (float)h->sum_w; ta.eps = (float)kEps64; ta.top_db = (float)h->p.top_db;
    ta.n_std = (float)h->p.n_std_thresh; ta.ddof = h->p.std_ddof; ta.mag = mag; ta.rowmax = rowmax; ta.thr = h->d_tthr;
    B200_LAUNCH(k_tgate_stats<>, dim3((unsigned)(Bn * kFW)), dim3(kTgWarps * 32), 0, st, ta);
    CK(h, cudaGetLastError());
    CK(h, cudaStreamSynchronize(st));
    h->tthr_units = (int)Bn;
    return B200GATE_OK;
}

// ---- the chunk grid of a run (base.py:167-226; b200gate_set_range) ---------------------------------------------------
// One computation serves run_core and the kept-mask layout, so the two cannot disagree on the units or their frames.
// torch surface (TorchGate.forward on whole rows): one unit per row, no padding, no ranges.
struct RunGrid {
    bool single_to = false;       // range mode 2: the reference's single padded chunk [0, a) (base.py:222)
    bool chunked = false;
    long long step = 0, n_chunks = 1, first = 0, count = 1, pad = 0, Lp = 0;
    int T = 0;                    // frames per unit
};

static int run_grid(b200gate_handle* h, long long N, RunGrid* rg) {
    const b200gate_params& p = h->p;
    const bool torch_rows = p.surface == B200GATE_SURFACE_TORCH;
    *rg = RunGrid{};
    rg->single_to = !torch_rows && h->range_mode == 2;
    if (rg->single_to && h->range_a > N) return fail(h, B200GATE_ERR_ARG, "range end %lld beyond the recording", h->range_a);
    rg->chunked = !torch_rows && !rg->single_to && p.chunk_size > 0 && N > p.chunk_size;
    rg->step = rg->chunked ? p.chunk_size : (rg->single_to ? h->range_a : N);
    rg->n_chunks = rg->chunked ? (N - 1) / p.chunk_size + 1 : 1;
    rg->count = rg->n_chunks;
    if (!torch_rows && h->range_mode == 1) {                 // a sub-range of the chunk grid
        if (!rg->chunked || h->range_b >= rg->n_chunks) return fail(h, B200GATE_ERR_ARG, "chunk range outside the chunk grid");
        rg->first = h->range_a;
        rg->count = h->range_b - h->range_a + 1;
    }
    rg->pad = torch_rows ? 0 : p.padding;                    // TorchGate.forward filters the whole row, no chunk padding
    rg->Lp = rg->step + 2 * rg->pad;
    if (rg->Lp / p.hop_length > 0x3fffffffLL) return fail(h, B200GATE_ERR_ARG, "problem too large");
    rg->T = h->generic ? (int)((rg->Lp + 2 * (h->g_W / 2) - h->g_W) / p.hop_length) + 1 : (int)(rg->Lp / p.hop_length) + 1;
    return B200GATE_OK;
}

// ---- kept masks (b200gate_mask_store_bytes / b200gate_set_mask_store / b200gate_adjoint) ----------------------------
// The layout of the masks a run keeps: every unit of the call in unit order, at a fixed size per unit, so that a batch's
// buffers sit at its unit offset whatever the batching.
struct MaskPlan {
    Geom g;                       // H, C, T, n_chunks, n_total, step, pad, Lp (u0 / n_units are per batch)
    long long U = 0, Ubase = 0;   // units of the call and its first unit
    size_t unit_bytes = 0;        // stationary, n_fft 1024: decision words [T][FW]; else the final mask [T][FPad] / [T][F]
    size_t off_rowflag = 0;       // stationary, n_fft 1024: the top_db row flags [U][FW] follow the decisions
    size_t bytes = 0;
};

static bool mask_family_ok(b200gate_handle* h) {
    if (h->p.surface != B200GATE_SURFACE_NUMPY) {
        fail(h, B200GATE_ERR_STATE, "kept masks and the adjoint are for the numpy surface (the torch surface's backward "
                                    "is b200gate_torch_apply_masks)");
        return false;
    }
    return true;
}

// the store layout of U units of T frames
static void mask_layout(const b200gate_handle* h, int T, long long U_, MaskPlan* mp) {
    const size_t U = (size_t)U_;
    if (h->generic) {
        mp->unit_bytes = (size_t)T * h->F * sizeof(double);
        mp->bytes = U * mp->unit_bytes;
    } else if (h->p.stationary) {
        mp->unit_bytes = (size_t)T * kFW * 4;
        mp->off_rowflag = (U * mp->unit_bytes + 255) / 256 * 256;
        mp->bytes = mp->off_rowflag + U * kFW * 4;
    } else {
        mp->unit_bytes = (size_t)T * (h->p.n_fft == kN2 ? kFPad2 : kFPad) * 4;
        mp->bytes = U * mp->unit_bytes;
    }
}

static int mask_plan(b200gate_handle* h, long long C, long long N, MaskPlan* mp) {
    if (!mask_family_ok(h)) return B200GATE_ERR_STATE;
    if (C <= 0 || N <= 0) return fail(h, B200GATE_ERR_ARG, "bad argument");
    RunGrid rg;
    const int rc = run_grid(h, N, &rg);
    if (rc) return rc;
    *mp = MaskPlan{};
    Geom& g = mp->g;
    g.H = h->p.hop_length; g.C = (int)C; g.n_total = N; g.n_chunks = (int)rg.n_chunks;
    g.step = rg.step; g.pad = rg.pad; g.Lp = rg.Lp; g.T = rg.T;
    mp->U = rg.count * C;
    mp->Ubase = rg.first * C;
    if (mp->Ubase + mp->U > 0x7fffffffLL) return fail(h, B200GATE_ERR_ARG, "problem too large");
    mask_layout(h, g.T, mp->U, mp);
    return B200GATE_OK;
}

// b200gate_run on input rows that hold only samples [in_first, N) (a stream's window, addressed through the virtual base
// `in` = window - in_first): the row stride then only has to cover that span.
static int run_core(b200gate_handle* h, const void* in, void* out, int dtype, int64_t C, int64_t N, int64_t in_stride,
                    int64_t out_stride, int is_device, void* stream, int64_t in_first) {
    if (!h || !in || !out || C <= 0 || N <= 0 || dtype_size(dtype) == 0) return fail(h, B200GATE_ERR_ARG, "bad argument");
    // torch_sem: TorchGate's arithmetic; torch_rows: TorchGate.forward on whole rows (no chunk grid, no ranges)
    const bool torch_sem = h->p.surface != B200GATE_SURFACE_NUMPY;
    const bool torch_rows = h->p.surface == B200GATE_SURFACE_TORCH;
    // torch.istft(center=True) length of an L-sample row: n_fft + hop (T - 1) minus n_fft/2 at both ends (torchgate.py:255-262)
    auto torch_len = [&](long long L) { return (L / h->p.hop_length) * h->p.hop_length + (h->p.n_fft & 1); };
    const int64_t No = torch_rows ? torch_len(N) : N;
    // In a range mode only samples [o_lo, o_hi) of a row are addressed, so `out` may be a virtual base
    // (slab - o_lo) over rows as short as the range: the stride check below uses the range length.
    if (in_stride < N - in_first || (out_stride < No && (torch_rows || h->range_mode == 0)))
        return fail(h, B200GATE_ERR_ARG, "row strides too small");
    if (torch_rows && N < 2 * h->p.win_length) return fail(h, B200GATE_ERR_ARG, "x must be bigger than %d", 2 * h->p.win_length);
    if (torch_sem && h->tthr_units > 1 && h->tthr_units != C)
        return fail(h, B200GATE_ERR_ARG, "xn has %d rows, x has %lld", h->tthr_units, (long long)C);
    if (h->p.stationary && !torch_sem && h->n_rec > 0)
        return fail(h, B200GATE_ERR_STATE, "per-recording thresholds are installed; they serve b200gate_run_rows only "
                    "(b200gate_set_noise_threshold or b200gate_noise_stats returns to one set)");
    if (h->p.stationary && !torch_sem && !h->have_thresh)
        return fail(h, B200GATE_ERR_STATE, "stationary gate: call b200gate_noise_stats first");
    cudaStream_t st = (cudaStream_t)stream;
    const b200gate_params& p = h->p;
    const size_t es = dtype_size(dtype);

    // ---- which part of the recording (base.py:167-226; b200gate_set_range) -----------------------------
    // range_mode 2: the reference's single padded chunk [0, a) inside a longer recording (base.py:222)
    RunGrid rg;
    {
        const int rc = run_grid(h, N, &rg);
        if (rc) return rc;
    }
    const bool chunked = rg.chunked;
    const long long step = rg.step;
    const long long n_chunks = rg.n_chunks;
    // the padded unit TorchGate filters: at least 2 win_length samples (torchgate.py:214-220); on the chunk grid its torch
    // output must hold the centre of a whole chunk (the reference's slice assignment fails otherwise, base.py:200-207)
    const long long unit_len = step + (torch_rows ? 0 : 2 * p.padding);
    if (torch_sem && !torch_rows && unit_len < 2 * p.win_length)
        return fail(h, B200GATE_ERR_ARG, "x must be bigger than %d", 2 * p.win_length);
    if (torch_sem && chunked && torch_len(unit_len) - p.padding < step)
        return fail(h, B200GATE_ERR_ARG, "could not broadcast: a padded chunk of %lld samples gives %lld torch output "
                    "samples, fewer than padding + chunk_size = %lld", unit_len, torch_len(unit_len), p.padding + step);
    h->stats = b200gate_stats{};
    long long launches = 0;
    if (!h->reuse_masks) h->masks_valid = false;
    // range_mode 1: a sub-range of the chunk grid
    const long long chunk_first = rg.first, chunk_count = rg.count;
    // samples written [o_lo, o_hi) and samples read [w_lo, w_hi)
    const long long o_lo = chunk_first * step;
    const long long o_hi = torch_rows ? No : std::min<long long>(N, (chunk_first + chunk_count) * step);
    const long long rpad = torch_rows ? 0 : p.padding;
    const long long w_lo = torch_rows ? 0 : std::max(0LL, o_lo - rpad);
    const long long w_hi = torch_rows ? N : std::min<long long>(N, o_hi + rpad);
    const long long Wn = w_hi - w_lo, On = o_hi - o_lo;
    if (out_stride < On) return fail(h, B200GATE_ERR_ARG, "output row stride %lld shorter than the range (%lld samples)",
                                     (long long)out_stride, On);

    // ---- where the kernels read / write ---------------------------------------------------------------
    // The n_fft = 1024 numpy-surface kernels are templated on the sample dtype: they read the caller's
    // float32 / int16 / float64 rows directly and cast on store (base.py:140, :218-226).  The 2048 family and
    // the torch surface run on float32 rows (other dtypes are converted at the edge).
    const bool generic = h->generic;
    // (the general family is templated on the sample type on both surfaces: float64 TorchGate input stays float64)
    const bool native = (!torch_sem && p.n_fft == kN) || generic;
    const int kdt = native ? dtype : B200GATE_F32;            // dtype the kernels see
    const size_t kes = dtype_size(kdt);
    const void* x = nullptr;
    void* y = nullptr;
    long long xs = in_stride, ys = out_stride;
    const bool direct = is_device && kdt == dtype;
    // Host input that the reference would chunk: stream it through the GPU slab by slab (H2D of slab k+1,
    // kernels of slab k and D2H of slab k-1 overlap on three streams) instead of staging the whole
    // recording -- the role of _read_chunk + the memmap write-back (base.py:130-187).
    const bool pipelined = !is_device && kdt == dtype && chunked && h->p.padding >= h->p.hop_length;
    if (direct || pipelined) {
        x = in;
        y = out;
    } else {
        // stage the window that is read / written; the kernels keep absolute sample indices through virtual
        // row bases (x - w_lo, y - o_lo)
        int rc;
        if ((rc = ensure(h, (void**)&h->d_in, &h->in_bytes, (size_t)C * Wn * kes))) return rc;
        if ((rc = ensure(h, (void**)&h->d_out, &h->out_bytes, (size_t)C * On * kes))) return rc;
        x = (const char*)h->d_in - (size_t)w_lo * kes;
        y = (char*)h->d_out - (size_t)o_lo * kes;
        xs = Wn;
        ys = On;
        if (kdt == dtype) {                                   // host rows
            CK(h, cudaMemcpy2DAsync(h->d_in, (size_t)Wn * es, (const char*)in + (size_t)w_lo * es, (size_t)in_stride * es,
                                    (size_t)Wn * es, (size_t)C, cudaMemcpyHostToDevice, st));
        } else {                                              // float32-only kernel family: convert at the edge
            const void* raw = (const char*)in + (size_t)w_lo * es;
            long long rs = in_stride;
            if (!is_device) {
                if ((rc = ensure(h, &h->d_raw, &h->raw_bytes, (size_t)C * std::max(Wn, On) * es))) return rc;
                CK(h, cudaMemcpy2DAsync(h->d_raw, (size_t)Wn * es, raw, (size_t)in_stride * es, (size_t)Wn * es, (size_t)C,
                                        cudaMemcpyHostToDevice, st));
                raw = h->d_raw;
                rs = Wn;
            }
            const int gr = grid_1d((long long)C * Wn, 256, h->num_sm * 16);
            if (dtype == B200GATE_I16)
                { auto kern_ = k_to_f32<short>; B200_LAUNCH(kern_, dim3(gr), dim3(256), 0, st, (const short*)raw, (float*)h->d_in, (long long)C, (long long)Wn, rs, (long long)Wn); }
            else
                { auto kern_ = k_to_f32<double>; B200_LAUNCH(kern_, dim3(gr), dim3(256), 0, st, (const double*)raw, (float*)h->d_in, (long long)C, (long long)Wn, rs, (long long)Wn); }
            ++launches;
        }
    }
    float h2d_ms = 0.f;
    cudaEvent_t evk0 = h->ev0, evk1 = h->ev1;

    // ---- geometry (base.py:167-226) -----------------------------------------------------------
    Geom g{};
    g.H = p.hop_length;
    g.C = (int)C;
    g.n_total = N;
    g.step = step;
    g.n_chunks = (int)n_chunks;
    g.pad = rg.pad;
    g.Lp = rg.Lp;
    g.T = rg.T;
    g.in_stride = xs;
    g.out_stride = ys;
    const long long U = chunk_count * C;
    const long long Ubase = chunk_first * C;               // first unit of the selected range
    if (Ubase + U > 0x7fffffffLL || g.Lp / g.H > 0x3fffffffLL) return fail(h, B200GATE_ERR_ARG, "problem too large");
    // kept masks (b200gate_set_mask_store): each batch's mask buffers are carved from the store at its unit offset
    MaskPlan kp{};
    const bool keep = h->keep_masks;
    if (keep) {                                            // (the layout of this very run's units and frames)
        mask_layout(h, g.T, U, &kp);
        if ((int64_t)kp.bytes > h->mask_store_bytes)
            return fail(h, B200GATE_ERR_ARG, "mask store of %lld bytes; this run keeps %zu", (long long)h->mask_store_bytes,
                        kp.bytes);
    }

    const int NFFT = p.n_fft;
    const bool two_k = NFFT == kN2 && !generic;
    const int FP = two_k ? kFPad2 : kFPad, FF = generic ? h->F : (two_k ? kF2 : kF);
    // frames whose masks k2 needs (same for every full chunk)
    const long long sig_len = (long long)(g.T - 1) * g.H + (generic ? (h->g_W & 1) : 0);
    long long jp_hi = std::min(g.pad + g.step, sig_len);
    int tf_lo = 0, tf_hi = 0;
    int h_lo = 0, h_hi = 0;
    if (jp_hi > g.pad) {
        h_lo = (int)((g.pad + NFFT / 2) / g.H);
        h_hi = (int)((jp_hi + NFFT / 2 + g.H - 1) / g.H);
        tf_lo = std::max(0, h_lo - 3) & ~1;          // even: k2 walks k1's (2j, 2j+1) frame pairs when spectra are cached
        tf_hi = std::min(h_hi, g.T);
    }
    const bool tail_zeros = !torch_sem && !generic && (g.pad + g.step > sig_len);   // (gk_ola writes the zeros itself)     // stationary.py:126 leaves the tail zero
    if (tail_zeros) {
        for (long long c = 0; c < C; ++c)
            CK(h, cudaMemsetAsync((char*)y + ((size_t)c * ys + (size_t)o_lo) * kes, 0, (size_t)On * kes, st));
    }

    // ---- workspace / batching ---------------------------------------------------------------------
    const bool stat = p.stationary != 0;
    // spectrum cache: k1 / k1n keep the packed spectrum of every frame pair so k2 does not re-transform
    const int zpairs = (g.T + 1) / 2;
    const bool use_zcache = !generic && !(p.path_flags & 2);
    // (n_fft 2048: one half-length spectrum per frame; n_fft 1024: one packed spectrum per frame pair)
    const size_t zunit = use_zcache ? (size_t)(two_k ? g.T : zpairs) * 1024 * sizeof(float2) : 0;
    // dual kernels (gate_dual.cuh): two channels of a chunk per warp -- stationary numpy-surface gate, even channel count.
    // Opt-in (path_flags bit 4): without packed FP32 instructions (sm_90) they are slower than one unit per warp.
    const bool use_dual = use_zcache && stat && !torch_sem && native && (C % 2 == 0) && (p.path_flags & 16);
    // stationary mask smoothing inside k2c_synthesize (kMaskBits*) for every filter the byte-lane arithmetic holds; the
    // separate smoothing kernel and the uint16 numerators in the workspace remain for the rest, for the dual and
    // re-transforming synthesis kernels, and on request (path_flags bit 8)
    const bool smooth_in_k2 = stat && use_zcache && !use_dual && !(p.path_flags & 256) &&
                              packed_smoothing_fits(p.n_grad_freq, p.n_grad_time);
    const size_t num_bytes = smooth_in_k2 ? 0 : (size_t)num_unit_stride(g.T) * 2;
    const size_t per_unit_2pass = (stat ? (size_t)g.T * kFW * 4 + (size_t)kFPad * 4 + (size_t)kFW * 4 + num_bytes + 64
                                        : 2 * (size_t)g.T * FP * 4 + 64) +
                                  (stat && torch_sem ? (size_t)g.T * kFPad * 4 + 2 * (size_t)kFPad * 4 : 0) + 2048;
    // general-geometry family: float64 spectrum, mask, scratch and synthesis frames of every unit
    const size_t g_tf = (size_t)g.T * (size_t)h->F, g_tw = (size_t)g.T * (size_t)h->g_W;
    const size_t per_unit_generic = g_tf * 16 + 2 * g_tf * 8 + g_tw * 8 + 2 * (size_t)h->F * 8 + 6 * 256;
    const size_t per_unit = generic ? per_unit_generic : per_unit_2pass + zunit;
    // default workspace: up to 24 GiB, never more than 70 % of what is free now (plus what this handle already holds)
    double limit = p.workspace_limit_bytes;
    if (!(limit > 0)) {
        limit = 24.0 * 1024 * 1024 * 1024;
        size_t free_b = 0, total_b = 0;
        if (cudaMemGetInfo(&free_b, &total_b) == cudaSuccess)
            limit = std::min(limit, 0.7 * ((double)free_b + (double)h->ws_bytes));
    }
    long long ub = (long long)std::max(1.0, floor(limit / (double)per_unit));
    ub = std::min(ub, U);
    if (use_dual) ub = std::max(2LL, ub & ~1LL);             // duals are units (2d, 2d+1) of a batch
    if (generic) ub = std::min(ub, 65535LL);                 // gk_* put the unit on gridDim.y
    // reserve the workspace now; if the device cannot give it (the caller's own tensors may fill HBM), halve the batch
    for (;;) {
        const size_t est = (size_t)ub * per_unit + ((size_t)8 << 20);
        if (ensure(h, (void**)&h->d_ws_buf, &h->ws_bytes, est) == B200GATE_OK) break;
        cudaGetLastError();
        long long nub = ub / 2;
        if (use_dual) nub &= ~1LL;
        if (nub < (use_dual ? 2 : 1)) return B200GATE_ERR_NOMEM;     // (message set by ensure)
        ub = nub;
    }
    if (!pipelined && ub < U) {
        // several batches: equal ones (a full batch followed by a small remainder would end every kernel of the remainder
        // in a partial wave); the slab pipeline sizes its batches itself below
        const long long nb = (U + ub - 1) / ub;
        long long eq = (U + nb - 1) / nb;
        if (use_dual) eq += eq & 1;
        ub = std::min(ub, std::max(eq, use_dual ? 2LL : 1LL));
    }
    long long slab_chunks = 0, slab_w = 0, slab_ow = 0;
    bool stage_in = false, stage_out = false;
    if (pipelined) {
        // ~256 MB of input per slab (large enough to keep the copy engines busy, small enough to pipeline), whole chunks, within the workspace limit
        long long slab_bytes = 256LL << 20;
        if (const char* e = getenv("B200GATE_SLAB_MB")) slab_bytes = std::max(1LL, atoll(e)) << 20;     // tuning knob
        slab_chunks = std::max(1LL, std::min<long long>(chunk_count, slab_bytes / std::max<long long>(1, C * g.step * (long long)es)));
        slab_chunks = std::max(1LL, std::min(slab_chunks, ub / C));
        if (ub < C) return fail(h, B200GATE_ERR_NOMEM, "workspace limit too small for one chunk of all channels");
        ub = slab_chunks * C;
        slab_w = slab_chunks * g.step + 2 * g.pad;
        slab_ow = slab_chunks * g.step;
        for (int i = 0; i < 2; ++i) {
            int rc;
            if ((rc = ensure(h, (void**)&h->d_slab_in[i], &h->slab_in_bytes[i], (size_t)C * slab_w * es))) return rc;
            if ((rc = ensure(h, (void**)&h->d_slab_out[i], &h->slab_out_bytes[i], (size_t)C * slab_ow * es))) return rc;
        }
        stage_in = !host_pointer_is_pinned(in);
        stage_out = !host_pointer_is_pinned(out);
        for (int i = 0; i < 2; ++i) {                  // pinned staging slabs for pageable caller memory (process-wide pool)
            if (stage_in && h->hp_in_bytes[i] < (size_t)C * slab_w * es) {
                g_pinned_pool.give(h->hp_in[i], h->hp_in_bytes[i]);
                h->hp_in[i] = g_pinned_pool.take((size_t)C * slab_w * es, &h->hp_in_bytes[i]);
                if (!h->hp_in[i]) { h->hp_in_bytes[i] = 0; return fail(h, B200GATE_ERR_NOMEM, "pinned staging slab (%zu bytes)", (size_t)C * slab_w * es); }
            }
            if (stage_out && h->hp_out_bytes[i] < (size_t)C * slab_ow * es) {
                g_pinned_pool.give(h->hp_out[i], h->hp_out_bytes[i]);
                h->hp_out[i] = g_pinned_pool.take((size_t)C * slab_ow * es, &h->hp_out_bytes[i]);
                if (!h->hp_out[i]) { h->hp_out_bytes[i] = 0; return fail(h, B200GATE_ERR_NOMEM, "pinned staging slab (%zu bytes)", (size_t)C * slab_ow * es); }
            }
        }
        if (const char* e = getenv("B200GATE_HOST_THREADS")) h->host_threads = std::max(1, atoi(e));
    }
    // carve the workspace into 256-byte aligned sub-buffers (vector stores need natural alignment)
    auto al = [](size_t v) { return (v + 255) / 256 * 256; };
    const size_t off_bits = 0;
    const size_t off_rowmax = off_bits + al((size_t)ub * g.T * kFW * 4);
    const size_t off_rowflag = off_rowmax + al((size_t)ub * kFPad * 4);
    const size_t off_num = off_rowflag + al((size_t)ub * kFW * 4);
    const size_t end_stat = off_num + al((size_t)ub * num_bytes);
    const size_t off_m0 = al((size_t)ub * g.T * FP * 4);
    const size_t end_nonstat = off_m0 + al((size_t)ub * g.T * FP * 4);
    // torch surface, stationary: the stationary buffers follow the dB spectrogram
    const size_t off_tdb = end_stat;
    const size_t off_trow = off_tdb + al((size_t)ub * g.T * kFPad * 4);
    const size_t off_tthr = off_trow + al((size_t)ub * kFPad * 4);
    const size_t end_tstat = off_tthr + al((size_t)ub * kFPad * 4);
    const size_t goff_M = al((size_t)ub * g_tf * 16);
    const size_t goff_tmp = goff_M + al((size_t)ub * g_tf * 8);
    const size_t goff_fr = goff_tmp + al((size_t)ub * g_tf * 8);
    const size_t goff_thr = goff_fr + al((size_t)ub * g_tw * 8);          // torch surface: per-row thresholds
    const size_t goff_rmax = goff_thr + al((size_t)ub * h->F * 8);         // per-(unit, bin) dB maxima (top_db floor)
    const size_t end_generic = goff_rmax + al((size_t)ub * h->F * 8);
    const size_t end_base = generic ? end_generic : (stat ? (torch_sem ? end_tstat : end_stat) : end_nonstat);
    const size_t off_z = al(end_base);
    const size_t end_all = off_z + al((size_t)ub * zunit);
    {
        int rc = ensure(h, (void**)&h->d_ws_buf, &h->ws_bytes, end_all);
        if (rc) return rc;
    }
    float* d_tdb = (float*)(h->d_ws_buf + off_tdb);
    float* d_trow = (float*)(h->d_ws_buf + off_trow);
    float* d_tthr_self = (float*)(h->d_ws_buf + off_tthr);
    float2* d_zcache = use_zcache ? (float2*)(h->d_ws_buf + off_z) : nullptr;
    unsigned* d_bits = (unsigned*)(h->d_ws_buf + off_bits);
    unsigned* d_rowmax = (unsigned*)(h->d_ws_buf + off_rowmax);
    unsigned* d_rowflag = (unsigned*)(h->d_ws_buf + off_rowflag);
    unsigned short* d_num = (unsigned short*)(h->d_ws_buf + off_num);
    float* d_mag = (float*)h->d_ws_buf;                        // non-stationary: |X|, later the final mask
    float* d_m0 = (float*)(h->d_ws_buf + off_m0);              //                 forward sweep / sigmoid mask

    CK(h, cudaMemsetAsync(h->d_cnt, 0, sizeof(Counters), st));
    const long long dbg_u = (h->dbg_chunk >= 0 && h->dbg_chunk < g.n_chunks && h->dbg_channel >= 0 && h->dbg_channel < C)
                                ? h->dbg_chunk * C + h->dbg_channel : -1;
    if (dbg_u >= 0) {
        if (h->dbg_T_alloc < (size_t)g.T) {
            if (h->d_dbg_spec) cudaFree(h->d_dbg_spec);
            if (h->d_dbg_mask) cudaFree(h->d_dbg_mask);
            if (h->d_dbg_bits) cudaFree(h->d_dbg_bits);
            const size_t fmax_ = (size_t)std::max(kF2, h->F);
            CK(h, cudaMalloc((void**)&h->d_dbg_spec, (size_t)g.T * fmax_ * 8));
            CK(h, cudaMalloc((void**)&h->d_dbg_mask, (size_t)g.T * fmax_ * 4));
            CK(h, cudaMalloc((void**)&h->d_dbg_bits, (size_t)g.T * std::max<size_t>(kFW, (fmax_ + 31) / 32) * 4));
            h->dbg_T_alloc = g.T;
        }
        CK(h, cudaMemsetAsync(h->d_dbg_spec, 0, (size_t)g.T * FF * 8, st));
        CK(h, cudaMemsetAsync(h->d_dbg_mask, 0, (size_t)g.T * FF * 4, st));
        h->dbg_T = g.T;
    } else {
        h->dbg_T = 0;
    }

    const Tables tb = device_tables(h);
    const int nf = p.n_grad_freq, nt = p.n_grad_time;
    const double D = (double)(nf + 1) * (nf + 1) * (nt + 1) * (nt + 1);
    const int resident = h->num_sm * 3;
    const size_t n_batches = (size_t)((U + ub - 1) / ub);
    while (h->stage_ev.size() < 4 * n_batches) {
        cudaEvent_t e;
        CK(h, cudaEventCreate(&e));
        h->stage_ev.push_back(e);
    }
    while (pipelined && h->pipe_ev.size() < 4 * n_batches) {
        cudaEvent_t e;
        CK(h, cudaEventCreate(&e));
        h->pipe_ev.push_back(e);
    }
    size_t bi = 0;
    int nu_prev = 0;
    long long prev_o0 = 0, prev_o1 = 0;
    std::future<void> out_task;
    cudaEventRecord(evk0, st);
    for (long long u0 = 0; u0 < U; u0 += ub, ++bi) {
        const int nu = (int)std::min(ub, U - u0);
        g.u0 = (int)(Ubase + u0);
        g.n_units = nu;
        if (keep && !generic) {
            char* ks = (char*)h->mask_store;
            if (stat) {
                d_bits = (unsigned*)(ks + (size_t)u0 * kp.unit_bytes);
                d_rowflag = (unsigned*)(ks + kp.off_rowflag + (size_t)u0 * kFW * 4);
            } else {
                d_mag = (float*)(ks + (size_t)u0 * kp.unit_bytes);
            }
        }
        const void* xb = x;
        void* yb = y;
        if (pipelined) {
            // slab = chunks [c0, c1): input window [w0, w1) of every channel, output [c0*step, o1)
            const long long c0 = (Ubase + u0) / C, c1 = c0 + nu / C;
            const long long w0 = std::max(0LL, c0 * g.step - g.pad), w1 = std::min<long long>(N, c1 * g.step + g.pad);
            const long long o0 = c0 * g.step, o1 = std::min<long long>(N, c1 * g.step);
            const int ib = (int)(bi & 1);
            // The head of this slab's window -- [w0, pw1), the 2*padding samples around the slab seam -- is already
            // on the device at the tail of the previous slab's buffer: copy it device-to-device and bring only
            // [pw1, w1) over PCIe, so every sample crosses the bus once.
            const long long pw1 = bi == 0 ? w0 : std::min<long long>(N, c0 * g.step + g.pad);
            if (bi >= 1) CK(h, cudaStreamWaitEvent(h->s_h2d, h->pipe_ev[4 * (bi - 1) + 3], 0));   // slab buffer free
            if (w1 > pw1) {
                const void* src = (const char*)in + (size_t)pw1 * es;
                size_t spitch = (size_t)in_stride * es;
                if (stage_in) {
                    // pageable rows: host threads copy them into this slab's pinned staging buffer (free once the H2D of
                    // slab bi-2 has completed), the copy engine takes them from there
                    if (bi >= 2) CK(h, cudaEventSynchronize(h->pipe_ev[4 * (bi - 2) + 0]));
                    parallel_rows_copy(h->hp_in[ib], (size_t)(w1 - pw1) * es, src, spitch, (size_t)(w1 - pw1) * es, (size_t)C,
                                       stage_out ? std::max(1, h->host_threads / 2) : h->host_threads);
                    src = h->hp_in[ib];
                    spitch = (size_t)(w1 - pw1) * es;
                }
                CK(h, cudaMemcpy2DAsync((char*)h->d_slab_in[ib] + (size_t)(pw1 - w0) * es, (size_t)slab_w * es, src, spitch,
                                        (size_t)(w1 - pw1) * es, (size_t)C, cudaMemcpyHostToDevice, h->s_h2d));
            }
            CK(h, cudaEventRecord(h->pipe_ev[4 * bi + 0], h->s_h2d));
            if (bi >= 1 && pw1 > w0) {
                const long long pw0 = std::max(0LL, (c0 - nu_prev / C) * g.step - g.pad);           // previous window start
                CK(h, cudaMemcpy2DAsync(h->d_slab_in[ib], (size_t)slab_w * es,
                                        (const char*)h->d_slab_in[ib ^ 1] + (size_t)(w0 - pw0) * es, (size_t)slab_w * es,
                                        (size_t)(pw1 - w0) * es, (size_t)C, cudaMemcpyDeviceToDevice, st));
            }
            CK(h, cudaEventRecord(h->pipe_ev[4 * bi + 3], st));     // previous buffer's tail consumed (and its kernels done)
            CK(h, cudaStreamWaitEvent(st, h->pipe_ev[4 * bi + 0], 0));
            if (bi >= 2) CK(h, cudaStreamWaitEvent(st, h->pipe_ev[4 * (bi - 2) + 2], 0));         // output buffer drained
            // virtual row bases so the kernels keep absolute sample indices
            xb = (const char*)h->d_slab_in[ib] - (size_t)w0 * es;
            yb = (char*)h->d_slab_out[ib] - (size_t)o0 * es;
            g.in_stride = slab_w;
            g.out_stride = slab_ow;
            (void)o1;
        }
        DebugTap dbg{};
        dbg.ul = (dbg_u >= Ubase + u0 && dbg_u < Ubase + u0 + nu) ? (int)(dbg_u - Ubase - u0) : -1;
        dbg.spec = h->d_dbg_spec;
        dbg.mask = h->d_dbg_mask;

        if (generic) {
            GGeom gg = generic_geom(h, g);
            if (torch_rows) gg.out_len = No;                // torch.istft length (torchgate.py:255-262)
            else if (torch_sem) gg.crop = torch_len(g.Lp) - g.pad;   // the unit's torch output from column pad on
            const GTables gt = generic_tables(h);
            const int F = h->F, W = h->g_W, FW = (F + 31) / 32;
            double2* gX = (double2*)h->d_ws_buf;
            double* gM = keep ? (double*)((char*)h->mask_store + (size_t)u0 * kp.unit_bytes) : (double*)(h->d_ws_buf + goff_M);
            double* gTmp = (double*)(h->d_ws_buf + goff_tmp);
            double* gFr = (double*)(h->d_ws_buf + goff_fr);
            const int thr_fft = generic_threads(generic_fft_len(h));
            const size_t smem_fft = (size_t)generic_fft_len(h) * sizeof(double2);
            const bool smooth = nf > 0 || nt > 0;
            if (dbg.ul >= 0) CK(h, cudaMemsetAsync(h->d_dbg_bits, 0, (size_t)g.T * FW * 4, st));
            cudaEventRecord(h->stage_ev[4 * bi + 0], st);
            B200_WITH_DTYPE(kdt, {
                GStftArgs<T> sa{};
                sa.gg = gg; sa.tb = gt; sa.x = (const T*)xb; sa.X = gX;
                auto kern_ = gk_stft<T>;
                B200_LAUNCH(kern_, dim3((unsigned)g.T, (unsigned)nu), dim3(thr_fft), smem_fft, st, sa); });
            const int gr_elem = grid_1d((long long)nu * g.T * F, 256, h->num_sm * 16);
            if (stat) {
                unsigned long long* gRmax = (unsigned long long*)(h->d_ws_buf + goff_rmax);
                CK(h, cudaMemsetAsync(gRmax, 0, (size_t)nu * F * 8, st));
                GDbArgs ba{};
                ba.n_units = nu; ba.T = g.T; ba.F = F; ba.eps = kEps64; ba.X = gX; ba.M = gM; ba.rowmax = gRmax;
                B200_LAUNCH(gk_db_rowmax, dim3((unsigned)((F + 63) / 64), (unsigned)((g.T + 63) / 64), (unsigned)nu), dim3(256), 0, st, ba);
                ++launches;
                GDecideArgs da{};
                da.n_units = nu; da.T = g.T; da.F = F; da.top_db = p.top_db; da.p = p.prop_decrease;
                da.thr = h->d_gthr; da.thr_units = 1; da.rowmax = gRmax;
                da.M = gM; da.dbg_ul = dbg.ul; da.FW = FW; da.dbg_bits = h->d_dbg_bits;
                if (torch_sem) {                        // torchgate.py:127-165: per-row statistics (own frames or xn's)
                    if (h->tthr_units > 0) {                // xn's rows are channels: unit (chunk, ch) reads row ch
                        da.thr = h->d_gtthr;
                        da.thr_units = h->tthr_units;
                        da.thr_rows = (int)C;
                        da.thr_u0 = g.u0;
                    } else {
                        double* gThr = (double*)(h->d_ws_buf + goff_thr);
                        GTStatArgs ta{};
                        ta.n_units = nu; ta.T = g.T; ta.F = F; ta.ddof = p.std_ddof; ta.eps = kEps64; ta.top_db = p.top_db;
                        ta.n_std = p.n_std_thresh; ta.X = gX; ta.scratch = gM; ta.thr = gThr;
                        B200_LAUNCH(gk_tstats, dim3((unsigned)(((long long)nu * F + 127) / 128)), dim3(128), 0, st, ta);
                        ++launches;
                        da.thr = gThr;
                        da.thr_units = nu;
                    }
                }
                B200_LAUNCH(gk_decide, dim3(gr_elem), dim3(256), 0, st, da);
            } else if (torch_sem) {                     // torchgate.py:168-198: moving-mean follower
                GMovArgs ma{};
                ma.n_units = nu; ma.T = g.T; ma.F = F; ma.n = std::max(1, p.n_movemean); ma.n_thresh = p.thresh_n_mult;
                ma.inv_temp = p.sigmoid_slope; ma.p = p.prop_decrease; ma.X = gX; ma.M = gM; ma.tmp = gTmp;
                B200_LAUNCH(gk_movmean, dim3((unsigned)(((long long)nu * F + 127) / 128)), dim3(128), 0, st, ma);
            } else {
                const double tfr = p.time_constant_s * p.sr / (double)p.hop_length;       // nonstationary.py:109-114
                B200_LAUNCH(gk_abs, dim3(gr_elem), dim3(256), 0, st, (const double2*)gX, (long long)nu * g.T * F, gM);
                GFollowArgs fa{};
                fa.n_units = nu; fa.T = g.T; fa.F = F; fa.b = (sqrt(1.0 + 4.0 * tfr * tfr) - 1.0) / (2.0 * tfr * tfr);
                fa.A = gM; fa.S = gTmp;
                B200_LAUNCH(gk_follow, dim3((unsigned)(((long long)nu * F + 127) / 128)), dim3(128), 0, st, fa);
                GSigmoidArgs ga{};
                ga.n = (long long)nu * g.T * F; ga.n_mult = p.thresh_n_mult; ga.slope = p.sigmoid_slope; ga.p = p.prop_decrease;
                ga.blend = smooth ? 0 : 1; ga.S = gTmp; ga.M = gM;
                B200_LAUNCH(gk_sigmoid, dim3(gr_elem), dim3(256), 0, st, ga);
                launches += 2;
            }
            cudaEventRecord(h->stage_ev[4 * bi + 1], st);
            launches += 2;
            if (smooth) {
                GSmoothArgs ga{};
                ga.n_units = nu; ga.T = g.T; ga.F = F; ga.nf = nf; ga.nt = nt; ga.inv_D = 1.0 / D; ga.p = p.prop_decrease;
                ga.blend = (stat || torch_sem) ? 0 : 1;                                  // stationary.py / torchgate.py blend before smoothing
                const int gr = grid_1d((long long)nu * g.T * F, 256, h->num_sm * 16);
                ga.src = gM; ga.dst = gTmp;
                B200_LAUNCH(gk_smooth_f, dim3(gr), dim3(256), 0, st, ga);
                ga.src = gTmp; ga.dst = gM;
                B200_LAUNCH(gk_smooth_t, dim3(gr), dim3(256), 0, st, ga);
                launches += 2;
            }
            cudaEventRecord(h->stage_ev[4 * bi + 2], st);
            {
                GIstftArgs ia{};
                ia.gg = gg; ia.tb = gt; ia.X = gX; ia.M = gM; ia.frames = gFr; ia.dbg_ul = dbg.ul;
                ia.dbg_spec = (float2*)h->d_dbg_spec; ia.dbg_mask = h->d_dbg_mask;
                B200_LAUNCH(gk_istft, dim3((unsigned)g.T, (unsigned)nu), dim3(thr_fft), smem_fft, st, ia);
                const long long out_max = torch_rows ? No : std::min<long long>(g.step, N);
                B200_WITH_DTYPE(kdt, {
                    GOlaArgs<T> oa{};
                    oa.gg = gg; oa.tb = gt; oa.frames = gFr; oa.y = (T*)yb;
                    auto kern_ = gk_ola<T>;
                    B200_LAUNCH(kern_, dim3((unsigned)grid_1d(out_max, 256, 1 << 16), (unsigned)nu), dim3(256), 0, st, oa); });
                (void)W;
                launches += 2;
            }
            cudaEventRecord(h->stage_ev[4 * bi + 3], st);
        } else if (stat) {
            if (torch_sem) {
                // TorchGate: |X| -> dB, per-row statistics over the row's own frames (or xn's), compare
                cudaEventRecord(h->stage_ev[4 * bi + 0], st);
                launch_k1n(g, tb, xb, kdt, h->reuse_masks ? nullptr : d_tdb, dbg, resident, st, d_zcache, tf_lo, tf_hi + 1);
                if (!h->reuse_masks) {
                TStatArgs ta{};
                ta.n_units = nu; ta.T = g.T; ta.in_scale = (float)h->sum_w; ta.eps = (float)kEps64;
                ta.top_db = (float)p.top_db; ta.n_std = (float)p.n_std_thresh; ta.ddof = p.std_ddof;
                ta.mag = d_tdb; ta.rowmax = d_trow; ta.thr = d_tthr_self;
                B200_LAUNCH(k_tgate_stats<>, dim3((unsigned)((long long)nu * kFW)), dim3(kTgWarps * 32), 0, st, ta);
                TBitsArgs ba{};
                ba.n_units = nu; ba.T = g.T; ba.top_db = (float)p.top_db; ba.db = d_tdb; ba.rowmax = d_trow; ba.bits = d_bits;
                if (h->tthr_units > 0) {
                    ba.thr = h->tthr_units == 1 ? h->d_tthr : h->d_tthr + (size_t)u0 * kFPad;
                    ba.thr_units = h->tthr_units == 1 ? 1 : nu;
                } else {
                    ba.thr = d_tthr_self;
                    ba.thr_units = nu;
                }
                B200_LAUNCH(k_tgate_bits<>, dim3((unsigned)((long long)nu * kFW)), dim3(kTgWarps * 32), 0, st, ba);
                CK(h, cudaMemsetAsync(d_rowflag, 0, (size_t)nu * kFW * 4, st));
                ++launches;
                }
            } else {
                CK(h, cudaMemsetAsync(d_rowmax, 0, (size_t)nu * kFPad * 4, st));
                cudaEventRecord(h->stage_ev[4 * bi + 0], st);
                // k1: frames per work item: enough items to fill the machine, runs long enough to amortise
                K1Args a1{};
                a1.g = g; a1.tb = tb; a1.x = xb; a1.bits = d_bits; a1.rowmax = d_rowmax; a1.cnt = h->d_cnt; a1.dbg = dbg;
                a1.zcache = d_zcache; a1.zpairs = zpairs;
                a1.z_lo = tf_lo; a1.z_hi = tf_hi + 1;           // k2 walks pairs (2j, 2j+1) of frames [tf_lo, tf_hi)
                {
                    long long want = (long long)h->num_sm * B200_K1_MINBLOCKS * kWarps * 4;
                    long long run = ((long long)nu * g.T + want - 1) / want;
                    run = std::max(8LL, std::min(64LL, run));
                    run += run & 1;
                    a1.run = (int)run;
                    a1.n_runs = (g.T + a1.run - 1) / a1.run;
                }
                const long long items1 = (long long)nu * a1.n_runs;
                const unsigned grid1 = (unsigned)grid_1d(items1, kWarps, h->num_sm * B200_K1_MINBLOCKS);
                // The analysis kernels below leave out the per-bin row maxima of the top_db floor and raise a device flag
                // when a frame could reach the floor; the row-maximum kernel k1_analyze<.., true> then runs behind them
                // (and returns at once otherwise).  path_flags bit 9: that kernel alone does the whole analysis.
                CK(h, cudaMemsetAsync(h->d_need_rowmax, 0, sizeof(unsigned), st));
                if (use_dual) {
                    // two channels per warp (gate_dual.cuh)
                    K1dArgs ad{};
                    ad.g = g; ad.tb = tb; ad.x = xb; ad.bits = d_bits; ad.zd = (float4*)d_zcache; ad.zpairs = zpairs;
                    ad.z_lo = tf_lo; ad.z_hi = tf_hi + 1; ad.cnt = h->d_cnt; ad.need_rowmax = h->d_need_rowmax;
                    if (getenv("B200GATE_DBG_NOCACHE_STORE")) ad.z_hi = 0;        // timing experiment only: results are wrong
                    ad.min_floor4 = (float)(4.0 * h->min_floor_amp * h->min_floor_amp);
                    ad.wa_max = h->wa_max; ad.dbg = dbg;
                    {
                        long long want = (long long)h->num_sm * kDualWarpsK1 * 4;
                        long long run = ((long long)(nu / 2) * g.T + want - 1) / want;
                        run = std::max(8LL, std::min(64LL, run));
                        run += run & 1;
                        ad.run = (int)run;
                        ad.n_runs = (g.T + ad.run - 1) / ad.run;
                    }
                    B200_WITH_DTYPE(kdt, { auto kern_ = k1d_analyze<8, T>;
                        B200_LAUNCH(kern_, dim3(grid_1d((long long)(nu / 2) * ad.n_runs, kDualWarpsK1, h->num_sm)),
                                    dim3(kDualWarpsK1 * 32), k1d_smem_bytes(), st, ad); });
                    ++launches;
                    a1.guard = h->d_need_rowmax;
                    a1.zcache = nullptr;
                } else if (!(p.path_flags & 512)) {
                    a1.need_rowmax = h->d_need_rowmax;
                    a1.min_floor4 = (float)(4.0 * h->min_floor_amp * h->min_floor_amp);
                    B200_WITH_DTYPE(kdt, { auto kern_ = k1_analyze<8, T>;
                        B200_LAUNCH(kern_, dim3(grid1), dim3(kThreads), k1_smem_floats() * 4, st, a1); });
                    ++launches;
                    a1.guard = h->d_need_rowmax;
                    a1.zcache = nullptr;
                }
                B200_WITH_DTYPE(kdt, { auto kern_ = k1_analyze<8, T, true>;
                    B200_LAUNCH(kern_, dim3(grid1), dim3(kThreads), k1_smem_floats() * 4, st, a1); });
                B200_LAUNCH(k_rowfloor, dim3(grid_1d((long long)nu * kFW, 256, 1 << 30)), dim3(256), 0, st, nu,
                            (const unsigned*)d_rowmax, (const float*)h->d_floor4, d_rowflag, h->d_cnt);
            }
            launches += 2;
            cudaEventRecord(h->stage_ev[4 * bi + 1], st);
            cudaEventRecord(h->stage_ev[4 * bi + 2], st);
            cudaEventRecord(h->stage_ev[4 * bi + 3], st);
            if (tf_hi > tf_lo) {
                SmoothArgs sa{};
                sa.n_units = nu; sa.T = g.T; sa.nf = nf; sa.nt = nt; sa.tf_lo = tf_lo; sa.tf_hi = tf_hi; sa.TT = 32;
                sa.bits = d_bits; sa.rowflag = d_rowflag; sa.num = d_num;
                if (smooth_in_k2) {
                    // k2c_synthesize smooths the decisions itself (they and the row flags stay in the workspace, so the
                    // reuse_masks backward gets the forward's masks too)
                } else if (h->reuse_masks) {
                    // the numerators of the last forward are still in d_num
                } else {
                    launch_stationary_numerators(h, sa, st);
                }
                cudaEventRecord(h->stage_ev[4 * bi + 2], st);
                K2Args a2{};
                a2.g = g; a2.tb = tb; a2.x = xb; a2.y = yb; a2.num = d_num; a2.zcache = d_zcache; a2.zpairs = zpairs;
                a2.pD = (float)(p.prop_decrease / D);
                a2.one_minus_p = (float)(1.0 - p.prop_decrease);
                a2.nt = nt;
                a2.dbg = dbg;
                {
                    const long long hops = h_hi - h_lo;
                    long long want = (long long)resident * kWarps * 4;
                    long long run = ((long long)nu * hops + want - 1) / want;
                    run = std::max(16LL, std::min(128LL, run));
                    run += run & 1;
                    a2.run = (int)run;
                    a2.n_runs = (int)((hops + a2.run - 1) / a2.run);
                }
                const long long items2 = (long long)nu * a2.n_runs;
                if (use_dual) {
                    K2dArgs ad{};
                    ad.g = g; ad.tb = tb; ad.y = yb; ad.num = d_num; ad.zd = (const float4*)d_zcache; ad.zpairs = zpairs;
                    ad.pD = a2.pD; ad.one_minus_p = a2.one_minus_p; ad.nt = nt; ad.dbg = dbg;
                    {
                        const long long hops = h_hi - h_lo;
                        long long want = (long long)h->num_sm * kDualWarpsK2 * 4;
                        long long run = ((long long)(nu / 2) * hops + want - 1) / want;
                        run = std::max(16LL, std::min(128LL, run));
                        run += run & 1;
                        ad.run = (int)run;
                        ad.n_runs = (int)((hops + ad.run - 1) / ad.run);
                    }
                    const long long itemsd = (long long)(nu / 2) * ad.n_runs;
                    if (ad.one_minus_p != 0.f) {
                        B200_WITH_DTYPE(kdt, { auto kern2 = k2d_synthesize<8, true, T>;
                            B200_LAUNCH(kern2, dim3(grid_1d(itemsd, kDualWarpsK2, h->num_sm)), dim3(kDualWarpsK2 * 32),
                                        k2d_smem_bytes(), st, ad); });
                    } else {
                        B200_WITH_DTYPE(kdt, { auto kern2 = k2d_synthesize<8, false, T>;
                            B200_LAUNCH(kern2, dim3(grid_1d(itemsd, kDualWarpsK2, h->num_sm)), dim3(kDualWarpsK2 * 32),
                                        k2d_smem_bytes(), st, ad); });
                    }
                } else if (smooth_in_k2) {         // cached spectra, smoothing of the decisions in the same kernel
                    a2.num = nullptr;
                    a2.bits = d_bits; a2.rowflag = d_rowflag;
                    set_k2c_smoothing_taps(a2, nf);
                    if (a2.one_minus_p != 0.f) {
                        B200_WITH_DTYPE(kdt, { auto kern2 = k2c_synthesize<8, kMaskBitsBlend, T>;
                            B200_LAUNCH(kern2, dim3(grid_1d(items2, kWarps, resident)), dim3(kThreads),
                                        k2c_smem_bytes<kMaskBitsBlend>(), st, a2); });
                    } else {
                        B200_WITH_DTYPE(kdt, { auto kern2 = k2c_synthesize<8, kMaskBits, T>;
                            B200_LAUNCH(kern2, dim3(grid_1d(items2, kWarps, resident)), dim3(kThreads),
                                        k2c_smem_bytes<kMaskBits>(), st, a2); });
                    }
                } else if (use_zcache) {           // spectra kept by k1: bulk-staged synthesis (gate_synth.cuh)
                    if (a2.one_minus_p != 0.f) {
                        B200_WITH_DTYPE(kdt, { auto kern2 = k2c_synthesize<8, kMaskU16Blend, T>;
                            B200_LAUNCH(kern2, dim3(grid_1d(items2, kWarps, resident)), dim3(kThreads),
                                        k2c_smem_bytes<kMaskU16Blend>(), st, a2); });
                    } else {
                        B200_WITH_DTYPE(kdt, { auto kern2 = k2c_synthesize<8, kMaskU16, T>;
                            B200_LAUNCH(kern2, dim3(grid_1d(items2, kWarps, resident)), dim3(kThreads),
                                        k2c_smem_bytes<kMaskU16>(), st, a2); });
                    }
                } else {
                    B200_WITH_DTYPE(kdt, { auto kern2 = k2_synthesize<8, false, T>;
                        B200_LAUNCH(kern2, dim3(grid_1d(items2, kWarps, resident)), dim3(kThreads),
                                    k2_smem_floats(g.H) * 4, st, a2); });
                }
                cudaEventRecord(h->stage_ev[4 * bi + 3], st);
                launches += 2;
            }
        } else {
            if (two_k) {
                Tables2 t2{};
                t2.wa2 = h->d_wa2; t2.ws2 = h->d_ws2; t2.tw = h->d_tw; t2.w2k = h->d_w2k; t2.invn2 = h->d_invn2;
                t2.ws_to_w = h->ws_to_w;
                const int res2 = h->num_sm * 2;
                cudaEventRecord(h->stage_ev[4 * bi + 0], st);
                K1n2Args a1{};
                a1.g = g; a1.tb = t2; a1.x = (const float*)xb; a1.mag = d_mag; a1.dbg = dbg;
                a1.zcache = d_zcache; a1.z_lo = tf_lo; a1.z_hi = tf_hi + 1;
                {
                    long long want = (long long)resident * kWarps * 4;
                    long long run = ((long long)nu * g.T + want - 1) / want;
                    a1.run = (int)std::max(4LL, std::min(64LL, run));
                    a1.n_runs = (g.T + a1.run - 1) / a1.run;
                }
                B200_LAUNCH(k1n_magnitude_2k, dim3(grid_1d((long long)nu * a1.n_runs, kWarps, resident)), dim3(kThreads),
                            k1n2_smem_floats() * 4, st, a1);
                cudaEventRecord(h->stage_ev[4 * bi + 1], st);
                IirArgs ia{};
                ia.n_units = nu; ia.T = g.T; ia.F = kF2; ia.FPad = kFPad2;
                {
                    const double tfr = p.time_constant_s * p.sr / (double)g.H;
                    ia.b = (sqrt(1.0 + 4.0 * tfr * tfr) - 1.0) / (2.0 * tfr * tfr);
                }
                ia.n_mult = (float)p.thresh_n_mult; ia.slope = (float)p.sigmoid_slope;
                ia.regen = iir_regen_ok(ia.b, g.T, p.path_flags);
                ia.mag = d_mag; ia.m0 = d_m0;
                B200_LAUNCH(k_iir_sigmoid<kFPad2>, dim3(grid_1d((long long)nu * kFPad2, 128, 1 << 30)), dim3(128), 0, st, ia);
                launches += 2;
                cudaEventRecord(h->stage_ev[4 * bi + 2], st);
                cudaEventRecord(h->stage_ev[4 * bi + 3], st);
                if (tf_hi > tf_lo) {
                    SmoothFArgs sa{};
                    sa.n_units = nu; sa.T = g.T; sa.nf = nf; sa.nt = nt; sa.tf_lo = tf_lo; sa.tf_hi = tf_hi; sa.TT = 16;
                    sa.F = kF2; sa.FPad = kFPad2;
                    sa.p = (float)p.prop_decrease; sa.one_minus_p = (float)(1.0 - p.prop_decrease);
                    sa.m0 = d_m0; sa.m2 = d_mag;
                    launch_smooth_float(sa, nf, nt, tf_lo, tf_hi, nu, p.path_flags, st);
                    cudaEventRecord(h->stage_ev[4 * bi + 2], st);
                    if (use_zcache) {                  // spectra kept by k1n: bulk-staged synthesis (gate_synth_2k.cuh)
                        K2c2Args ac{};
                        ac.g = g; ac.tb = t2; ac.y = (float*)yb; ac.fmask = d_mag; ac.zcache = d_zcache; ac.dbg = dbg;
                        const long long hops = h_hi - h_lo;
                        long long want = (long long)h->num_sm * kK2c2Warps * 4;
                        long long run = ((long long)nu * hops + want - 1) / want;
                        ac.run = (int)std::max(16LL, std::min(128LL, run));
                        ac.n_runs = (int)((hops + ac.run - 1) / ac.run);
                        B200_LAUNCH(k2c_synthesize_2k, dim3(grid_1d((long long)nu * ac.n_runs, kK2c2Warps, h->num_sm)),
                                    dim3(kK2c2Warps * 32), k2c2_smem_bytes(), st, ac);
                    } else {
                    K22Args a2{};
                    a2.g = g; a2.tb = t2; a2.x = (const float*)xb; a2.y = (float*)yb; a2.fmask = d_mag; a2.dbg = dbg;
                    {
                        const long long hops = h_hi - h_lo;
                        long long want = (long long)res2 * kWarps * 4;
                        long long run = ((long long)nu * hops + want - 1) / want;
                        a2.run = (int)std::max(16LL, std::min(128LL, run));
                        a2.n_runs = (int)((hops + a2.run - 1) / a2.run);
                    }
                    B200_LAUNCH(k2_synthesize_2k<>, dim3(grid_1d((long long)nu * a2.n_runs, kWarps, res2)), dim3(kThreads),
                                k22_smem_floats() * 4, st, a2);
                    }
                    cudaEventRecord(h->stage_ev[4 * bi + 3], st);
                    launches += 2;
                }
            } else {
                cudaEventRecord(h->stage_ev[4 * bi + 0], st);
                launch_k1n(g, tb, xb, kdt, h->reuse_masks ? nullptr : d_mag, dbg, resident, st, d_zcache, tf_lo, tf_hi + 1);
                cudaEventRecord(h->stage_ev[4 * bi + 1], st);
                if (h->reuse_masks) {
                    // the final masks of the last forward are still in d_mag
                } else if (torch_sem) {
                    TMovArgs ma{};
                    ma.n_units = nu; ma.T = g.T; ma.n_movemean = p.n_movemean; ma.n_thresh = (float)p.thresh_n_mult;
                    ma.inv_temp = (float)p.sigmoid_slope; ma.p = (float)p.prop_decrease; ma.mag = d_mag; ma.m0 = d_m0;
                    B200_LAUNCH(k_tgate_movmean<>, dim3(grid_1d((long long)nu * kFPad, 128, 1 << 30)), dim3(128), 0, st, ma);
                } else {
                    IirArgs ia{};
                    ia.n_units = nu; ia.T = g.T; ia.F = kF; ia.FPad = kFPad;
                    {
                        const double tfr = p.time_constant_s * p.sr / (double)g.H;        // nonstationary.py:109-114
                        ia.b = (sqrt(1.0 + 4.0 * tfr * tfr) - 1.0) / (2.0 * tfr * tfr);
                    }
                    ia.n_mult = (float)p.thresh_n_mult; ia.slope = (float)p.sigmoid_slope;
                    ia.regen = iir_regen_ok(ia.b, g.T, p.path_flags);
                    ia.mag = d_mag; ia.m0 = d_m0;
                    B200_LAUNCH(k_iir_sigmoid<kFPad>, dim3(grid_1d((long long)nu * kFPad, 128, 1 << 30)), dim3(128), 0, st, ia);
                }
                launches += 2;
                cudaEventRecord(h->stage_ev[4 * bi + 2], st);
                cudaEventRecord(h->stage_ev[4 * bi + 3], st);
                if (tf_hi > tf_lo) {
                    SmoothFArgs sa{};
                    sa.n_units = nu; sa.T = g.T; sa.nf = nf; sa.nt = nt; sa.tf_lo = tf_lo; sa.tf_hi = tf_hi; sa.TT = 32;
                    sa.F = kF; sa.FPad = kFPad;
                    sa.p = torch_sem ? 1.0f : (float)p.prop_decrease;
                    sa.one_minus_p = torch_sem ? 0.0f : (float)(1.0 - p.prop_decrease);
                    sa.m0 = d_m0; sa.m2 = d_mag;
                    if (h->reuse_masks) {
                        // masks of the last forward
                    } else {
                        launch_smooth_float(sa, nf, nt, tf_lo, tf_hi, nu, p.path_flags, st);
                    }
                    cudaEventRecord(h->stage_ev[4 * bi + 2], st);
                    K2Args a2{};
                    a2.g = g; a2.tb = tb; a2.x = xb; a2.y = yb; a2.fmask = d_mag; a2.zcache = d_zcache; a2.zpairs = zpairs;
                    a2.nt = nt;
                    a2.dbg = dbg;
                    {
                        const long long hops = h_hi - h_lo;
                        long long want = (long long)resident * kWarps * 4;
                        long long run = ((long long)nu * hops + want - 1) / want;
                        run = std::max(16LL, std::min(128LL, run));
                        run += run & 1;
                        a2.run = (int)run;
                        a2.n_runs = (int)((hops + a2.run - 1) / a2.run);
                    }
                    if (use_zcache) {
                        B200_WITH_DTYPE(kdt, { auto kern2 = k2c_synthesize<8, kMaskF32, T>;
                            B200_LAUNCH(kern2, dim3(grid_1d((long long)nu * a2.n_runs, kWarps, resident)), dim3(kThreads),
                                        k2c_smem_bytes<kMaskF32>(), st, a2); });
                    } else {
                        B200_WITH_DTYPE(kdt, { auto kern2 = k2_synthesize<8, true, T>;
                            B200_LAUNCH(kern2, dim3(grid_1d((long long)nu * a2.n_runs, kWarps, resident)), dim3(kThreads),
                                        k2_smem_floats(g.H) * 4, st, a2); });
                    }
                    cudaEventRecord(h->stage_ev[4 * bi + 3], st);
                    launches += 2;
                }
            }
        }
        if (dbg.ul >= 0 && stat && !generic) {
            // tapped mask words with the row floor folded in, as the smoothing kernel consumes them
            std::vector<unsigned> fl(kFW);
            CK(h, cudaStreamSynchronize(st));
            CK(h, cudaMemcpy(fl.data(), d_rowflag + (size_t)dbg.ul * kFW, kFW * 4, cudaMemcpyDeviceToHost));
            std::vector<unsigned> bb((size_t)g.T * kFW);
            CK(h, cudaMemcpy(bb.data(), d_bits + (size_t)dbg.ul * g.T * kFW, bb.size() * 4, cudaMemcpyDeviceToHost));
            for (size_t i = 0; i < bb.size(); ++i) bb[i] |= fl[i % kFW];
            CK(h, cudaMemcpy(h->d_dbg_bits, bb.data(), bb.size() * 4, cudaMemcpyHostToDevice));
        }
        CK(h, cudaGetLastError());
        if (pipelined) {
            const long long c0 = (Ubase + u0) / C, c1 = c0 + nu / C;
            const long long o0 = c0 * g.step, o1 = std::min<long long>(N, c1 * g.step);
            const int ib = (int)(bi & 1);
            const void* d2h_src = h->d_slab_out[ib];
            CK(h, cudaEventRecord(h->pipe_ev[4 * bi + 1], st));
            CK(h, cudaStreamWaitEvent(h->s_d2h, h->pipe_ev[4 * bi + 1], 0));
            if (stage_out) {
                if (out_task.valid()) out_task.get();       // slab bi-2 has left this staging buffer
                // pageable result rows: D2H into this slab's pinned staging buffer (its previous content, slab bi-2, was
                // copied out by the host below), then the host threads move slab bi-1 -- whose D2H has had a whole slab of
                // kernel time -- into the caller's array
                CK(h, cudaMemcpy2DAsync(h->hp_out[ib], (size_t)(o1 - o0) * es, d2h_src, (size_t)slab_ow * es,
                                        (size_t)(o1 - o0) * es, (size_t)C, cudaMemcpyDeviceToHost, h->s_d2h));
                CK(h, cudaEventRecord(h->pipe_ev[4 * bi + 2], h->s_d2h));
                if (bi >= 1) {
                    // runs beside the next slab's copy-in (joined before that slab's D2H is enqueued into this staging buffer's twin)
                    cudaEvent_t evd = h->pipe_ev[4 * (bi - 1) + 2];
                    void* dstp = (char*)out + (size_t)prev_o0 * es;
                    const void* srcp = h->hp_out[ib ^ 1];
                    const size_t wbytes = (size_t)(prev_o1 - prev_o0) * es, dp = (size_t)out_stride * es;
                    const int nth = std::max(1, h->host_threads / 2), dev_now = h->device;
                    out_task = std::async(std::launch::async, [evd, dstp, srcp, wbytes, dp, C, nth, dev_now]() {
                        cudaSetDevice(dev_now);
                        cudaEventSynchronize(evd);
                        parallel_rows_copy(dstp, dp, srcp, wbytes, wbytes, (size_t)C, nth, 1);
                    });
                }
                prev_o0 = o0; prev_o1 = o1;
            } else {
                CK(h, cudaMemcpy2DAsync((char*)out + (size_t)o0 * es, (size_t)out_stride * es, d2h_src, (size_t)slab_ow * es,
                                        (size_t)(o1 - o0) * es, (size_t)C, cudaMemcpyDeviceToHost, h->s_d2h));
                CK(h, cudaEventRecord(h->pipe_ev[4 * bi + 2], h->s_d2h));
            }
            nu_prev = nu;
        }
    }
    cudaEventRecord(evk1, st);
    if (pipelined) {
        CK(h, cudaStreamSynchronize(h->s_d2h));
        CK(h, cudaStreamSynchronize(h->s_h2d));
        if (out_task.valid()) out_task.get();
        if (stage_out && bi >= 1)                      // the last slab's rows
            parallel_rows_copy((char*)out + (size_t)prev_o0 * es, (size_t)out_stride * es, h->hp_out[(bi - 1) & 1],
                               (size_t)(prev_o1 - prev_o0) * es, (size_t)(prev_o1 - prev_o0) * es, (size_t)C, h->host_threads, 1);
        if (getenv("B200GATE_TRACE")) {                       // slab timeline (ms since the first launch) on stderr
            CK(h, cudaStreamSynchronize(st));
            for (size_t b = 0; b < n_batches; ++b) {
                float t[4] = {0, 0, 0, 0};
                for (int i = 0; i < 4; ++i) cudaEventElapsedTime(&t[i], evk0, h->pipe_ev[4 * b + i]);
                fprintf(stderr, "slab %3zu  h2d_done %8.3f  seam_done %8.3f  kernels_done %8.3f  d2h_done %8.3f\n", b, t[0],
                        t[3], t[1], t[2]);
            }
        }
    }

    // ---- results back -------------------------------------------------------------------------------
    if (!direct && !pipelined) {
        void* out_w = (char*)out + (size_t)o_lo * es;             // first written sample of row 0
        if (kdt == dtype) {
            CK(h, cudaMemcpy2DAsync(out_w, (size_t)out_stride * es, h->d_out, (size_t)On * es, (size_t)On * es, (size_t)C,
                                    cudaMemcpyDeviceToHost, st));
        } else {
            int rc;
            if ((rc = ensure(h, &h->d_raw, &h->raw_bytes, (size_t)C * std::max(Wn, On) * es))) return rc;
            const int gr = grid_1d((long long)C * On, 256, h->num_sm * 16);
            void* dst = is_device ? out_w : h->d_raw;
            const long long ds = is_device ? out_stride : On;
            if (dtype == B200GATE_I16)
                { auto kern_ = k_from_f32<short>; B200_LAUNCH(kern_, dim3(gr), dim3(256), 0, st, (const float*)h->d_out, (short*)dst, (long long)C, (long long)On, (long long)On, ds); }
            else
                { auto kern_ = k_from_f32<double>; B200_LAUNCH(kern_, dim3(gr), dim3(256), 0, st, (const float*)h->d_out, (double*)dst, (long long)C, (long long)On, (long long)On, ds); }
            ++launches;
            if (!is_device)
                CK(h, cudaMemcpy2DAsync(out_w, (size_t)out_stride * es, h->d_raw, (size_t)On * es, (size_t)On * es, (size_t)C,
                                        cudaMemcpyDeviceToHost, st));
        }
    }
    CK(h, cudaGetLastError());

    // ---- stats: the counters travel to pinned host memory behind the kernels; a device-pointer run returns
    // here with everything enqueued (b200gate_get_stats waits for it), host-pointer runs return finished -----
    CK(h, cudaMemcpyAsync(h->h_cnt, h->d_cnt, sizeof(Counters), cudaMemcpyDeviceToHost, st));
    CK(h, cudaEventRecord(h->ev_done, st));
    h->stats.units = U;
    h->stats.frames = U * g.T;
    h->stats.kernel_launches = launches;
    h->stats.fused_path = 0;
    h->stats_pending = true;
    if (torch_sem && !generic && !two_k && n_batches == 1 && !h->reuse_masks) {
        h->masks_valid = true; h->masks_C = C; h->masks_N = N;
        h->masks_rows_n.clear();
    }
    h->pend_batches = n_batches;
    if (keep) {
        for (size_t i = h->kept.size(); i-- > 0;)
            if (h->kept[i].store == h->mask_store) h->kept.erase(h->kept.begin() + (long)i);
        if (h->kept.size() >= 64) h->kept.erase(h->kept.begin());
        h->kept.push_back({h->mask_store, (long long)C, (long long)N, h->range_a, h->range_b, h->range_mode, kp.bytes});
    }
    if (!direct) {                               // host buffers: the result must be in `out` on return
        const int rc = resolve_stats(h);
        if (rc) return rc;
    }
    h->stats.last_h2d_ms = h2d_ms;
    return B200GATE_OK;
}

int b200gate_run(b200gate_handle* h, const void* in, void* out, int dtype, int64_t C, int64_t N, int64_t in_stride,
                 int64_t out_stride, int is_device, void* stream) {
    if (h && h->s_open) return fail(h, B200GATE_ERR_STATE, "a stream is open on this handle (b200gate_stream_finish first)");
    if (h && h->ts_open) return fail(h, B200GATE_ERR_STATE, kTsOpen);
    if (h) h->keep_masks = h->mask_store != nullptr;
    const int rc = run_core(h, in, out, dtype, C, N, in_stride, out_stride, is_device, stream, 0);
    if (h) h->keep_masks = false;
    return rc;
}

// ---- b200gate_run_rows: rows of different lengths in one call ---------------------------------------------------------
// Every row is a recording of its own: it is cut into units exactly as run_grid() cuts a [1][n] recording (one padded
// chunk of n + 2 pad samples when n <= chunk_size, else chunks of chunk_size + 2 pad), the units of all rows form one
// table (UnitDesc) and the ROWS instantiations of the default kernels of run_core walk it.  Per-unit buffers have the
// pitch of the call's longest unit; everything that run_core derives from T or Lp is derived per unit here.
int b200gate_run_rows(b200gate_handle* h, const b200gate_row* rows, int64_t n_rows, int dtype, int is_device, void* stream) {
    if (!h || !rows || n_rows <= 0 || dtype_size(dtype) == 0) return fail(h, B200GATE_ERR_ARG, "bad argument");
    if (h->s_open) return fail(h, B200GATE_ERR_STATE, "a stream is open on this handle (b200gate_stream_finish first)");
    if (h->ts_open) return fail(h, B200GATE_ERR_STATE, kTsOpen);
    const b200gate_params& p = h->p;
    // torch: TorchGate.forward on each row (one unit per row: no chunk grid, no padding, torch.istft output length)
    const bool torch = p.surface == B200GATE_SURFACE_TORCH;
    if (p.surface != B200GATE_SURFACE_NUMPY && !torch)
        return fail(h, B200GATE_ERR_STATE, "b200gate_run_rows is for the numpy and torch surfaces");
    if (h->mask_store) return fail(h, B200GATE_ERR_STATE, "b200gate_run_rows keeps no masks (b200gate_set_mask_store(NULL) first)");
    if (h->range_mode != 0) return fail(h, B200GATE_ERR_STATE, "b200gate_run_rows runs whole rows (b200gate_set_range(0) first)");
    if (h->generic || p.n_fft != kN)                            // (a big smoothing filter also makes the handle generic)
        return fail(h, B200GATE_ERR_ARG, "b200gate_run_rows runs the n_fft 1024 kernels: it needs n_fft = win_length = 1024, "
                    "hop_length = 256 and smoothing extents (%d, %d) within their 16-bit numerators ((nf + 1)^2 (nt + 1)^2 "
                    "<= 65535, at most 64 a side)", p.n_grad_freq, p.n_grad_time);
    if (p.path_flags != 0) return fail(h, B200GATE_ERR_ARG, "b200gate_run_rows runs the default kernel selection (path_flags = 0)");
    if (torch && dtype != B200GATE_F32) return fail(h, B200GATE_ERR_ARG, "b200gate_run_rows: the torch surface runs float32 rows");
    const bool stat = p.stationary != 0;
    const int nf = p.n_grad_freq, nt = p.n_grad_time;
    // stationary: smoothing in the synthesis kernel where the byte lanes hold the filter; on the torch surface the
    // numerator kernel k_smooth_generic takes the other extents
    const bool smooth_in_k2 = packed_smoothing_fits(nf, nt);
    if (stat && !torch && !smooth_in_k2)
        return fail(h, B200GATE_ERR_ARG, "b200gate_run_rows: stationary smoothing extents (%d, %d) beyond the in-synthesis smoothing", nf, nt);
    if (!stat && !((nf >= 1 && nf <= 12 && smoothb_smem_bytes(kFPad, nt) <= 200 * 1024) || smooths_smem_bytes(kFPad, nf, nt) <= 200 * 1024))
        return fail(h, B200GATE_ERR_ARG, "b200gate_run_rows: smoothing extents (%d, %d) beyond the streaming smoothing kernels", nf, nt);
    // per-recording thresholds (b200gate_set_noise_threshold_rows): every unit reads its recording's rows of the tables
    const bool perrec = stat && !torch && h->n_rec > 0;
    if (stat && !torch && !h->have_thresh && !perrec)
        return fail(h, B200GATE_ERR_STATE, "stationary gate: call b200gate_noise_stats first");
    if (torch && h->tthr_units > 1 && h->tthr_units != n_rows)
        return fail(h, B200GATE_ERR_ARG, "xn has %d rows, the call has %lld", h->tthr_units, (long long)n_rows);
    cudaStream_t st = (cudaStream_t)stream;
    const size_t es = dtype_size(dtype);
    const int H = p.hop_length;
    const long long pad = torch ? 0 : p.padding, cs = torch ? 0 : p.chunk_size;
    const bool reuse = h->reuse_masks;                          // b200gate_torch_apply_masks_rows
    // torch.istft(center=True) length of an n-sample row (torchgate.py:255-262)
    auto out_len = [&](long long n) { return torch ? (n / H) * H + (p.n_fft & 1) : n; };

    // ---- the unit table -------------------------------------------------------------------------------------
    const char *in_lo = nullptr, *in_hi = nullptr, *out_lo = nullptr, *out_hi = nullptr;    // spans covering the rows
    size_t row_bytes = 0;
    long long U = 0;
    for (int64_t r = 0; r < n_rows; ++r) {
        const b200gate_row& rw = rows[r];
        if (!rw.in || !rw.out || rw.n <= 0 || rw.channels <= 0)
            return fail(h, B200GATE_ERR_ARG, "row %lld: null pointer, no samples or no channels", (long long)r);
        if (torch && rw.n < 2 * p.win_length)
            return fail(h, B200GATE_ERR_ARG, "row %lld: x must be bigger than %d", (long long)r, 2 * p.win_length);
        const char *a = (const char*)rw.in, *b = (const char*)rw.out;
        const size_t nb = (size_t)rw.n * es, nbo = (size_t)out_len(rw.n) * es;
        if (a < b + nbo && b < a + nb) return fail(h, B200GATE_ERR_ARG, "row %lld: out aliases in", (long long)r);
        const long long Lp = (cs > 0 && rw.n > cs ? cs : rw.n) + 2 * pad;
        if (Lp / H > 0x3fffffffLL) return fail(h, B200GATE_ERR_ARG, "problem too large");
        U += cs > 0 && rw.n > cs ? (rw.n - 1) / cs + 1 : 1;
        if (!in_lo || a < in_lo) in_lo = a;
        if (!in_hi || a + nb > in_hi) in_hi = a + nb;
        if (!out_lo || b < out_lo) out_lo = b;
        if (!out_hi || b + nbo > out_hi) out_hi = b + nbo;
        row_bytes += nb;
    }
    if (U > 0x7fffffffLL) return fail(h, B200GATE_ERR_ARG, "problem too large");
    if (perrec) {                  // rows group into recordings in order: `channels` consecutive rows of equal n and channels
        long long groups = 0;
        for (int64_t r = 0; r < n_rows; r += rows[r].channels, ++groups) {
            const int64_t k = rows[r].channels;
            if (k > n_rows - r)
                return fail(h, B200GATE_ERR_ARG, "row %lld starts a recording of %lld channels, %lld rows follow",
                            (long long)r, (long long)k, (long long)(n_rows - r));
            for (int64_t j = r + 1; j < r + k; ++j)
                if (rows[j].n != rows[r].n || rows[j].channels != k)
                    return fail(h, B200GATE_ERR_ARG, "row %lld: the channels of the recording from row %lld differ in n "
                                "or channels", (long long)j, (long long)r);
        }
        if (groups != h->n_rec)
            return fail(h, B200GATE_ERR_ARG, "the rows form %lld recordings, %d have thresholds", groups, h->n_rec);
    }
    // host rows travel as the two spans that cover them, one copy each way: they must come packed in one buffer
    const size_t in_span = (size_t)(in_hi - in_lo), out_span = (size_t)(out_hi - out_lo);
    if (!is_device && std::max(in_span, out_span) > 2 * row_bytes + 4096 * (size_t)n_rows)
        return fail(h, B200GATE_ERR_ARG, "host rows must lie in one buffer (they are copied as the span that covers them)");
    const size_t tbytes = (size_t)U * sizeof(UnitDesc);
    if (!h->ev_units) CK(h, cudaEventCreateWithFlags(&h->ev_units, cudaEventDisableTiming));
    else CK(h, cudaEventSynchronize(h->ev_units));             // the last call's table has left hp_units
    if (h->hp_units_bytes < tbytes) {
        g_pinned_pool.give(h->hp_units, h->hp_units_bytes);
        h->hp_units =(UnitDesc*)g_pinned_pool.take(tbytes, &h->hp_units_bytes);
        if (!h->hp_units) { h->hp_units_bytes = 0; return fail(h, B200GATE_ERR_NOMEM, "pinned unit table (%zu bytes)", tbytes); }
    }
    {
        int rc;
        if ((rc = ensure(h, &h->d_units, &h->units_bytes, tbytes))) return rc;
        if (!is_device) {
            if ((rc = ensure(h, (void**)&h->d_in, &h->in_bytes, in_span))) return rc;
            if ((rc = ensure(h, (void**)&h->d_out, &h->out_bytes, out_span))) return rc;
        }
    }
    double b_iir = 0.0;
    if (!stat) {
        const double tfr = p.time_constant_s * p.sr / (double)H;                    // nonstationary.py:109-114
        b_iir = (sqrt(1.0 + 4.0 * tfr * tfr) - 1.0) / (2.0 * tfr * tfr);
    }
    // frames whose masks the synthesis needs: [tf_lo, tf_hi) with the first one shared by every unit (run_core)
    const int h_lo = (int)((pad + kN / 2) / H);
    const int tf_lo = std::max(0, h_lo - 3) & ~1;
    int T_max = 0, tf_hi_max = 0;
    long long n_runs2 = 0;                                      // synthesis work items per unit: the most any unit needs
    const int resident = h->num_sm * 3;
    long long frames = 0;
    std::vector<long long> zero_units;                          // units whose centre reaches past their istft output
    {
        long long u = 0;
        int rec = -1;                                           // perrec: the row's recording
        for (int64_t r = 0, left = 0; r < n_rows; ++r, --left) {
            const b200gate_row& rw = rows[r];
            if (left == 0) { ++rec; left = rw.channels; }
            const bool chunked = cs > 0 && rw.n > cs;
            const long long step = chunked ? cs : rw.n, nch = chunked ? (rw.n - 1) / cs + 1 : 1;
            const void* x = is_device ? rw.in : (const void*)((const char*)h->d_in + ((const char*)rw.in - in_lo));
            void* y = is_device ? rw.out : (void*)((char*)h->d_out + ((const char*)rw.out - out_lo));
            for (long long ic = 0; ic < nch; ++ic, ++u) {
                UnitDesc& d = h->hp_units[u];
                d.x = x; d.y = y; d.n_total = rw.n;
                d.i1 = ic * step - pad;
                d.Lp = step + 2 * pad;
                d.o_lo = ic * step;
                d.o_hi = std::min<long long>(rw.n, (ic + 1) * step);
                d.T = (int)(d.Lp / H) + 1;
                const long long sig_len = (long long)(d.T - 1) * H;
                const long long jp_hi = std::min(pad + step, sig_len);
                int h_hi = 0;
                d.tf_hi = 0;
                if (jp_hi > pad) {
                    h_hi = (int)((jp_hi + kN / 2 + H - 1) / H);
                    d.tf_hi = std::min(h_hi, d.T);
                }
                d.regen = stat || torch ? 0 : iir_regen_ok(b_iir, d.T, 0);
                if (perrec) d.rec = rec;
                // stationary.py:126 leaves the tail zero (a torch row's output ends with its istft length)
                if (!torch && pad + step > sig_len) zero_units.push_back(u);
                {   // hops per synthesis work item: run_core's choice for a [channels][n] recording in one workspace batch
                    const long long hops = std::max(0, h_hi - h_lo), want = (long long)resident * kWarps * 4;
                    long long run = std::max(16LL, std::min(128LL, (nch * rw.channels * hops + want - 1) / want));
                    run += run & 1;
                    d.run = (int)run;
                    n_runs2 = std::max(n_runs2, (hops + run - 1) / run);
                }
                T_max = std::max(T_max, d.T);
                tf_hi_max = std::max(tf_hi_max, d.tf_hi);
                frames += d.T;
            }
        }
    }
    h->stats = b200gate_stats{};
    if (!reuse) h->masks_valid = false;
    long long launches = 0;
    CK(h, cudaMemcpyAsync(h->d_units, h->hp_units, tbytes, cudaMemcpyHostToDevice, st));
    CK(h, cudaEventRecord(h->ev_units, st));
    const UnitDesc* d_units = (const UnitDesc*)h->d_units;
    if (!is_device) CK(h, cudaMemcpyAsync(h->d_in, in_lo, in_span, cudaMemcpyHostToDevice, st));
    if (!is_device && torch) CK(h, cudaMemsetAsync(h->d_out, 0, out_span, st));     // (the span's bytes between rows)
    for (long long u : zero_units) {
        const UnitDesc& d = h->hp_units[u];
        CK(h, cudaMemsetAsync((char*)d.y + (size_t)d.o_lo * es, 0, (size_t)(d.o_hi - d.o_lo) * es, st));
    }

    // ---- workspace: run_core's per-unit buffers at the pitch of the longest unit ---------------------------------------
    Geom g{};
    g.H = H; g.C = 1; g.T = T_max; g.pad = pad;
    const int zpairs = (T_max + 1) / 2;
    const size_t zunit = (size_t)zpairs * 1024 * sizeof(float2);
    // torch surface, stationary: the dB spectrogram, its row maxima and self thresholds, and the numerators of
    // k_smooth_generic when the synthesis kernel cannot smooth the decisions itself
    const size_t num_bytes = smooth_in_k2 ? 0 : (size_t)num_unit_stride(T_max) * 2;
    const size_t per_unit = (stat ? (size_t)T_max * kFW * 4 + (size_t)kFPad * 4 + (size_t)kFW * 4 + 64
                                  : 2 * (size_t)T_max * kFPad * 4 + 64) +
                            (stat && torch ? num_bytes + (size_t)T_max * kFPad * 4 + 2 * (size_t)kFPad * 4 : 0) + 2048 + zunit;
    double limit = p.workspace_limit_bytes;
    if (!(limit > 0)) {
        limit = 24.0 * 1024 * 1024 * 1024;
        size_t free_b = 0, total_b = 0;
        if (cudaMemGetInfo(&free_b, &total_b) == cudaSuccess)
            limit = std::min(limit, 0.7 * ((double)free_b + (double)h->ws_bytes));
    }
    // the backward applies the masks the forward left in its one workspace batch: same units, same layout
    long long ub = reuse ? U : std::min(U, (long long)std::max(1.0, floor(limit / (double)per_unit)));
    for (;;) {                                                  // as run_core: halve the batch if the device cannot give it
        if (ensure(h, (void**)&h->d_ws_buf, &h->ws_bytes, (size_t)ub * per_unit + ((size_t)8 << 20)) == B200GATE_OK) break;
        cudaGetLastError();
        if (ub / 2 < 1) return B200GATE_ERR_NOMEM;
        ub /= 2;
    }
    if (ub < U) {                                               // equal batches
        const long long nb = (U + ub - 1) / ub;
        ub = std::min(ub, std::max((U + nb - 1) / nb, 1LL));
    }
    auto al = [](size_t v) { return (v + 255) / 256 * 256; };
    const size_t off_rowmax = al((size_t)ub * T_max * kFW * 4);
    const size_t off_rowflag = off_rowmax + al((size_t)ub * kFPad * 4);
    const size_t off_num = off_rowflag + al((size_t)ub * kFW * 4);
    const size_t off_tdb = off_num + al((size_t)ub * num_bytes);
    const size_t off_trow = off_tdb + al((size_t)ub * T_max * kFPad * 4);
    const size_t off_tthr = off_trow + al((size_t)ub * kFPad * 4);
    const size_t end_stat = torch ? off_tthr + al((size_t)ub * kFPad * 4) : off_num;
    const size_t off_m0 = al((size_t)ub * T_max * kFPad * 4);
    const size_t end_nonstat = off_m0 + al((size_t)ub * T_max * kFPad * 4);
    const size_t off_z = al(stat ? end_stat : end_nonstat);
    {
        const int rc = ensure(h, (void**)&h->d_ws_buf, &h->ws_bytes, off_z + al((size_t)ub * zunit));
        if (rc) return rc;
    }
    unsigned* d_bits = (unsigned*)h->d_ws_buf;
    unsigned* d_rowmax = (unsigned*)(h->d_ws_buf + off_rowmax);
    unsigned* d_rowflag = (unsigned*)(h->d_ws_buf + off_rowflag);
    unsigned short* d_num = (unsigned short*)(h->d_ws_buf + off_num);
    float* d_tdb = (float*)(h->d_ws_buf + off_tdb);
    float* d_trow = (float*)(h->d_ws_buf + off_trow);
    float* d_tthr_self = (float*)(h->d_ws_buf + off_tthr);
    float* d_mag = (float*)h->d_ws_buf;
    float* d_m0 = (float*)(h->d_ws_buf + off_m0);
    float2* d_zcache = (float2*)(h->d_ws_buf + off_z);

    CK(h, cudaMemsetAsync(h->d_cnt, 0, sizeof(Counters), st));
    h->dbg_T = 0;
    const Tables tb = device_tables(h);
    const double D = (double)(nf + 1) * (nf + 1) * (nt + 1) * (nt + 1);
    const size_t n_batches = (size_t)((U + ub - 1) / ub);
    while (h->stage_ev.size() < 4 * n_batches) {
        cudaEvent_t e;
        CK(h, cudaEventCreate(&e));
        h->stage_ev.push_back(e);
    }
    DebugTap dbg{};
    dbg.ul = -1;
    const long long hops = n_runs2;                             // (> 0: some unit has output hops)
    size_t bi = 0;
    cudaEventRecord(h->ev0, st);
    for (long long u0 = 0; u0 < U; u0 += ub, ++bi) {
        const int nu = (int)std::min(ub, U - u0);
        g.u0 = (int)u0;
        g.n_units = nu;
        // frames per analysis work item, sized as in run_core (the synthesis work items: UnitDesc::run)
        long long want = (long long)(stat ? h->num_sm * B200_K1_MINBLOCKS : resident) * kWarps * 4;
        long long run1 = std::max(8LL, std::min(64LL, ((long long)nu * T_max + want - 1) / want));
        run1 += run1 & 1;
        const int n_runs1 = (int)((T_max + run1 - 1) / run1);
        K2Args a2{};
        a2.g = g; a2.tb = tb; a2.zcache = d_zcache; a2.zpairs = zpairs; a2.nt = nt; a2.dbg = dbg; a2.units = d_units;
        a2.n_runs = (int)n_runs2;
        const unsigned grid2 = (unsigned)grid_1d((long long)nu * a2.n_runs, kWarps, resident);
        cudaEventRecord(h->stage_ev[4 * bi + 0], st);
        K1nArgs an{};                                           // k1n_magnitude: the torch surface and the non-stationary gate
        an.g = g; an.tb = tb; an.dbg = dbg; an.zcache = d_zcache; an.zpairs = zpairs;
        an.z_lo = tf_lo; an.z_hi = tf_hi_max + 1; an.units = d_units;
        an.run = (int)run1; an.n_runs = n_runs1;
        const unsigned grid1n = (unsigned)grid_1d((long long)nu * n_runs1, kWarps, resident);
        if (stat && torch) {
            // TorchGate (run_core): |X| -> dB, statistics over each row's own frames (or xn's), compare; the backward
            // (reuse) re-transforms only and synthesises with the decisions / numerators the forward left in the workspace
            an.mag = reuse ? nullptr : d_tdb;
            { auto kern_ = k1n_magnitude<8, float, true>;
              B200_LAUNCH(kern_, dim3(grid1n), dim3(kThreads), k1n_smem_floats() * 4, st, an); }
            ++launches;
            if (!reuse) {
                TStatArgs ta{};
                ta.n_units = nu; ta.T = T_max; ta.in_scale = (float)h->sum_w; ta.eps = (float)kEps64;
                ta.top_db = (float)p.top_db; ta.n_std = (float)p.n_std_thresh; ta.ddof = p.std_ddof;
                ta.mag = d_tdb; ta.rowmax = d_trow; ta.thr = d_tthr_self; ta.units = d_units + u0;
                { auto kern_ = k_tgate_stats<true>;
                  B200_LAUNCH(kern_, dim3((unsigned)((long long)nu * kFW)), dim3(kTgWarps * 32), 0, st, ta); }
                TBitsArgs ba{};
                ba.n_units = nu; ba.T = T_max; ba.top_db = (float)p.top_db; ba.db = d_tdb; ba.rowmax = d_trow; ba.bits = d_bits;
                ba.units = d_units + u0;
                if (h->tthr_units > 0) {                        // xn: one row for every unit, or row r for unit r
                    ba.thr = h->tthr_units == 1 ? h->d_tthr : h->d_tthr + (size_t)u0 * kFPad;
                    ba.thr_units = h->tthr_units == 1 ? 1 : nu;
                } else {
                    ba.thr = d_tthr_self;
                    ba.thr_units = nu;
                }
                { auto kern_ = k_tgate_bits<true>;
                  B200_LAUNCH(kern_, dim3((unsigned)((long long)nu * kFW)), dim3(kTgWarps * 32), 0, st, ba); }
                CK(h, cudaMemsetAsync(d_rowflag, 0, (size_t)nu * kFW * 4, st));
                launches += 2;
                if (!smooth_in_k2 && tf_hi_max > tf_lo) {
                    SmoothArgs sa{};
                    sa.n_units = nu; sa.T = T_max; sa.nf = nf; sa.nt = nt; sa.tf_lo = tf_lo; sa.tf_hi = tf_hi_max; sa.TT = 32;
                    sa.bits = d_bits; sa.rowflag = d_rowflag; sa.num = d_num; sa.units = d_units + u0;
                    auto kern_ = k_smooth_generic<true>;
                    B200_LAUNCH(kern_, dim3((tf_hi_max - tf_lo + sa.TT - 1) / sa.TT, nu), dim3(256),
                                smooth_smem_bytes(sa.TT, nf, nt), st, sa);
                    ++launches;
                }
            }
            cudaEventRecord(h->stage_ev[4 * bi + 1], st);
            cudaEventRecord(h->stage_ev[4 * bi + 2], st);
            if (hops > 0) {
                a2.pD = (float)(p.prop_decrease / D);
                a2.one_minus_p = (float)(1.0 - p.prop_decrease);
                const bool blend = a2.one_minus_p != 0.f;
                if (smooth_in_k2) {
                    a2.bits = d_bits; a2.rowflag = d_rowflag;
                    set_k2c_smoothing_taps(a2, nf);
                    auto kern2 = blend ? k2c_synthesize<8, kMaskBitsBlend, float, true> : k2c_synthesize<8, kMaskBits, float, true>;
                    B200_LAUNCH(kern2, dim3(grid2), dim3(kThreads), k2c_smem_bytes<kMaskBits>(), st, a2);
                } else {
                    a2.num = d_num;
                    auto kern2 = blend ? k2c_synthesize<8, kMaskU16Blend, float, true> : k2c_synthesize<8, kMaskU16, float, true>;
                    B200_LAUNCH(kern2, dim3(grid2), dim3(kThreads), k2c_smem_bytes<kMaskU16>(), st, a2);
                }
                ++launches;
            }
        } else if (stat) {
            CK(h, cudaMemsetAsync(d_rowmax, 0, (size_t)nu * kFPad * 4, st));
            CK(h, cudaMemsetAsync(h->d_need_rowmax, 0, sizeof(unsigned), st));
            K1Args a1{};
            a1.g = g; a1.tb = tb; a1.bits = d_bits; a1.rowmax = d_rowmax; a1.cnt = h->d_cnt; a1.dbg = dbg;
            a1.zcache = d_zcache; a1.zpairs = zpairs; a1.z_lo = tf_lo; a1.z_hi = tf_hi_max + 1; a1.units = d_units;
            a1.run = (int)run1; a1.n_runs = n_runs1;
            a1.need_rowmax = h->d_need_rowmax;
            a1.min_floor4 = (float)(4.0 * h->min_floor_amp * h->min_floor_amp);
            const unsigned grid1 = (unsigned)grid_1d((long long)nu * n_runs1, kWarps, h->num_sm * B200_K1_MINBLOCKS);
            const dim3 grid_rf(grid_1d((long long)nu * kFW, 256, 1 << 30));
            if (perrec) {                                       // each unit reads its recording's rows of the tables
                a1.tb = rec_tables(h, tb);
                B200_WITH_DTYPE(dtype, { auto kern_ = k1_analyze<8, T, false, true, true>;
                    B200_LAUNCH(kern_, dim3(grid1), dim3(kThreads), k1_smem_floats() * 4, st, a1); });
                a1.guard = h->d_need_rowmax;
                a1.zcache = nullptr;
                B200_WITH_DTYPE(dtype, { auto kern_ = k1_analyze<8, T, true, true, true>;
                    B200_LAUNCH(kern_, dim3(grid1), dim3(kThreads), k1_smem_floats() * 4, st, a1); });
                B200_LAUNCH(k_rowfloor_rec, grid_rf, dim3(256), 0, st, nu, d_units + u0, (const unsigned*)d_rowmax,
                            a1.tb.floor4, d_rowflag, h->d_cnt);
            } else {
                B200_WITH_DTYPE(dtype, { auto kern_ = k1_analyze<8, T, false, true>;
                    B200_LAUNCH(kern_, dim3(grid1), dim3(kThreads), k1_smem_floats() * 4, st, a1); });
                a1.guard = h->d_need_rowmax;                    // the row-maximum fallback, as in run_core
                a1.zcache = nullptr;
                B200_WITH_DTYPE(dtype, { auto kern_ = k1_analyze<8, T, true, true>;
                    B200_LAUNCH(kern_, dim3(grid1), dim3(kThreads), k1_smem_floats() * 4, st, a1); });
                B200_LAUNCH(k_rowfloor, grid_rf, dim3(256), 0, st, nu,
                            (const unsigned*)d_rowmax, (const float*)h->d_floor4, d_rowflag, h->d_cnt);
            }
            launches += 3;
            cudaEventRecord(h->stage_ev[4 * bi + 1], st);
            cudaEventRecord(h->stage_ev[4 * bi + 2], st);
            if (hops > 0) {
                a2.pD = (float)(p.prop_decrease / D);
                a2.one_minus_p = (float)(1.0 - p.prop_decrease);
                a2.bits = d_bits; a2.rowflag = d_rowflag;
                set_k2c_smoothing_taps(a2, nf);
                if (a2.one_minus_p != 0.f) {
                    B200_WITH_DTYPE(dtype, { auto kern2 = k2c_synthesize<8, kMaskBitsBlend, T, true>;
                        B200_LAUNCH(kern2, dim3(grid2), dim3(kThreads), k2c_smem_bytes<kMaskBitsBlend>(), st, a2); });
                } else {
                    B200_WITH_DTYPE(dtype, { auto kern2 = k2c_synthesize<8, kMaskBits, T, true>;
                        B200_LAUNCH(kern2, dim3(grid2), dim3(kThreads), k2c_smem_bytes<kMaskBits>(), st, a2); });
                }
                ++launches;
            }
        } else {
            an.mag = reuse ? nullptr : d_mag;
            B200_WITH_DTYPE(dtype, { auto kern_ = k1n_magnitude<8, T, true>;
                B200_LAUNCH(kern_, dim3(grid1n), dim3(kThreads), k1n_smem_floats() * 4, st, an); });
            cudaEventRecord(h->stage_ev[4 * bi + 1], st);
            if (reuse) {
                // the final masks of the forward are still in d_mag
            } else if (torch) {                                 // torchgate.py:168-198: moving-mean follower
                TMovArgs ma{};
                ma.n_units = nu; ma.T = T_max; ma.n_movemean = p.n_movemean; ma.n_thresh = (float)p.thresh_n_mult;
                ma.inv_temp = (float)p.sigmoid_slope; ma.p = (float)p.prop_decrease; ma.mag = d_mag; ma.m0 = d_m0;
                ma.units = d_units + u0;
                auto kern_ = k_tgate_movmean<true>;
                B200_LAUNCH(kern_, dim3(grid_1d((long long)nu * kFPad, 128, 1 << 30)), dim3(128), 0, st, ma);
            } else {
                IirArgs ia{};
                ia.n_units = nu; ia.T = T_max; ia.F = kF; ia.FPad = kFPad; ia.b = b_iir;
                ia.n_mult = (float)p.thresh_n_mult; ia.slope = (float)p.sigmoid_slope;
                ia.mag = d_mag; ia.m0 = d_m0; ia.units = d_units + u0;    // (regen: each unit's own, UnitDesc::regen)
                { auto kern_ = k_iir_sigmoid<kFPad, true>;
                  B200_LAUNCH(kern_, dim3(grid_1d((long long)nu * kFPad, 128, 1 << 30)), dim3(128), 0, st, ia); }
            }
            launches += reuse ? 1 : 2;
            if (tf_hi_max > tf_lo && !reuse) {
                SmoothFArgs sa{};
                sa.n_units = nu; sa.T = T_max; sa.nf = nf; sa.nt = nt; sa.tf_lo = tf_lo; sa.tf_hi = tf_hi_max; sa.TT = 32;
                sa.F = kF; sa.FPad = kFPad;
                // the torch surface blends before the smoothing (in k_tgate_movmean, torchgate.py:241)
                sa.p = torch ? 1.0f : (float)p.prop_decrease; sa.one_minus_p = torch ? 0.0f : (float)(1.0 - p.prop_decrease);
                sa.m0 = d_m0; sa.m2 = d_mag; sa.units = d_units + u0;
                launch_smooth_float<true>(sa, nf, nt, tf_lo, tf_hi_max, nu, 0, st);      // (extents checked on entry)
                ++launches;
            }
            cudaEventRecord(h->stage_ev[4 * bi + 2], st);
            if (hops > 0 && tf_hi_max > tf_lo) {
                a2.fmask = d_mag;
                B200_WITH_DTYPE(dtype, { auto kern2 = k2c_synthesize<8, kMaskF32, T, true>;
                    B200_LAUNCH(kern2, dim3(grid2), dim3(kThreads), k2c_smem_bytes<kMaskF32>(), st, a2); });
                ++launches;
            }
        }
        cudaEventRecord(h->stage_ev[4 * bi + 3], st);
        CK(h, cudaGetLastError());
    }
    cudaEventRecord(h->ev1, st);
    if (!is_device) CK(h, cudaMemcpyAsync((void*)out_lo, h->d_out, out_span, cudaMemcpyDeviceToHost, st));
    CK(h, cudaMemcpyAsync(h->h_cnt, h->d_cnt, sizeof(Counters), cudaMemcpyDeviceToHost, st));
    CK(h, cudaEventRecord(h->ev_done, st));
    h->stats.units = U;
    h->stats.frames = frames;
    h->stats.kernel_launches = launches;
    h->stats_pending = true;
    h->pend_batches = n_batches;
    if (torch && n_batches == 1 && !reuse) {      // the masks stay in the workspace for b200gate_torch_apply_masks_rows
        h->masks_valid = true; h->masks_C = 0; h->masks_N = 0;
        h->masks_rows_n.resize((size_t)n_rows);
        for (int64_t r = 0; r < n_rows; ++r) h->masks_rows_n[(size_t)r] = rows[r].n;
    }
    if (!is_device) {                            // host rows: the results must be in place on return
        const int rc = resolve_stats(h);
        if (rc) return rc;
    }
    return B200GATE_OK;
}

int b200gate_mask_store_bytes(b200gate_handle* h, int64_t C, int64_t N, int64_t* bytes) {
    if (!h || !bytes) return B200GATE_ERR_ARG;
    MaskPlan kp{};
    const int rc = mask_plan(h, C, N, &kp);
    if (rc) return rc;
    *bytes = (int64_t)kp.bytes;
    return B200GATE_OK;
}

int b200gate_set_mask_store(b200gate_handle* h, void* store, int64_t bytes) {
    if (!h) return B200GATE_ERR_ARG;
    if (store && !mask_family_ok(h)) return B200GATE_ERR_STATE;
    if (store && bytes <= 0) return fail(h, B200GATE_ERR_ARG, "mask store of %lld bytes", (long long)bytes);
    h->mask_store = store;
    h->mask_store_bytes = store ? bytes : 0;
    return B200GATE_OK;
}

}  // extern "C"

namespace {
template <typename T>
int adjoint_impl(b200gate_handle* h, const MaskPlan& kp, const char* store, const T* gin, T* grad, long long g_stride,
                 long long grad_stride, cudaStream_t st) {
    const b200gate_params& p = h->p;
    const bool generic = h->generic, stat = p.stationary != 0;
    const bool two_k = !generic && p.n_fft == kN2;             // float32 rows only (as run_core converts at the edge)
    const long long C = kp.g.C, N = kp.g.n_total, U = kp.U, Ubase = kp.Ubase;
    Geom g = kp.g;
    g.in_stride = g_stride;
    g.out_stride = grad_stride;
    const void* gk = gin;                                      // g as the synthesis kernel reads it
    if (two_k && sizeof(T) != sizeof(float)) {
        // the n_fft 2048 kernels read float32 rows: g's centre samples [o_lo, o_hi) go through the staging buffer
        const long long o_lo = (Ubase / C) * g.step, o_hi = std::min<long long>(N, (Ubase + U) / C * g.step);
        const long long On = o_hi - o_lo;
        int rc;
        if ((rc = ensure(h, (void**)&h->d_in, &h->in_bytes, (size_t)C * On * sizeof(float)))) return rc;
        { auto kern_ = k_to_f32<T>;
          B200_LAUNCH(kern_, dim3(grid_1d(C * On, 256, h->num_sm * 16)), dim3(256), 0, st, gin + o_lo, (float*)h->d_in, C, On,
                      g_stride, On); }
        gk = (const float*)h->d_in - o_lo;
        g.in_stride = On;
    }
    // every sample of grad is written: zeros where no unit of the call reads the input
    if (C == 1 || grad_stride == N)
        CK(h, cudaMemsetAsync(grad, 0, (size_t)C * N * sizeof(T), st));
    else
        for (long long c = 0; c < C; ++c) CK(h, cudaMemsetAsync(grad + c * grad_stride, 0, (size_t)N * sizeof(T), st));
    // frames whose masks the synthesis applies (run_core's tf_lo / tf_hi and output hops h_lo / h_hi of a full chunk)
    const int NFFT = p.n_fft;
    const long long sig_len = (long long)(g.T - 1) * g.H + (generic ? (h->g_W & 1) : 0);
    const long long jp_hi = std::min(g.pad + g.step, sig_len);
    if (jp_hi <= g.pad) return B200GATE_OK;                  // no unit writes a sample: the gradient is zero
    const int h_lo = (int)((g.pad + NFFT / 2) / g.H), h_hi = (int)((jp_hi + NFFT / 2 + g.H - 1) / g.H);
    const int tf_lo = std::max(0, h_lo - 3) & ~1, tf_hi = std::min(h_hi, g.T);
    // per-unit workspace: the adjoint's span [0, Lp), plus the numerators (stationary) or the spectra and synthesis
    // frames (general family)
    auto al = [](size_t v) { return (v + 255) / 256 * 256; };
    const size_t g_tf = (size_t)g.T * (size_t)h->F, g_tw = (size_t)g.T * (size_t)h->g_W;
    const size_t num_bytes = (!generic && stat) ? (size_t)num_unit_stride(g.T) * 2 : 0;
    const size_t adj_es = generic ? sizeof(double) : sizeof(float);
    const size_t per_unit = generic ? g_tf * 16 + g_tw * 8 + (size_t)g.Lp * 8 + 3 * 256
                                    : num_bytes + (size_t)g.Lp * 4 + 2 * 256;
    double limit = p.workspace_limit_bytes;
    if (!(limit > 0)) {
        limit = 24.0 * 1024 * 1024 * 1024;
        size_t free_b = 0, total_b = 0;
        if (cudaMemGetInfo(&free_b, &total_b) == cudaSuccess)
            limit = std::min(limit, 0.7 * ((double)free_b + (double)h->ws_bytes));
    }
    long long ub = std::min<long long>(U, (long long)std::max(1.0, floor(limit / (double)per_unit)));
    if (generic) ub = std::min(ub, 65535LL);
    for (;;) {
        if (ensure(h, (void**)&h->d_ws_buf, &h->ws_bytes, (size_t)ub * per_unit + ((size_t)8 << 20)) == B200GATE_OK) break;
        cudaGetLastError();
        if (ub / 2 < 1) return B200GATE_ERR_NOMEM;           // (message set by ensure)
        ub /= 2;
    }
    if (ub < U) {                                            // equal batches, as run_core
        const long long nb = (U + ub - 1) / ub;
        ub = std::min(ub, (U + nb - 1) / nb);
    }
    char* ws = h->d_ws_buf;
    const size_t off_a = generic ? al((size_t)ub * g_tf * 16) : 0;          // generic: spectra, then frames
    const size_t off_adj = generic ? off_a + al((size_t)ub * g_tw * 8) : al((size_t)ub * num_bytes);
    const long long adj_pitch = g.Lp;
    const int resident = h->num_sm * 3;
    const Tables tb = device_tables(h);
    const int nf = p.n_grad_freq, nt = p.n_grad_time;
    const double D = (double)(nf + 1) * (nf + 1) * (nt + 1) * (nt + 1);
    for (long long u0 = 0; u0 < U; u0 += ub) {
        const int nu = (int)std::min(ub, U - u0);
        g.u0 = (int)(Ubase + u0);
        g.n_units = nu;
        if (generic) {
            const GGeom gg = generic_geom(h, g);
            const GTables gt = generic_tables(h);
            double2* gX = (double2*)ws;
            double* gFr = (double*)(ws + off_a);
            double* adj = (double*)(ws + off_adj);
            const int thr_fft = generic_threads(generic_fft_len(h));
            const size_t smem_fft = (size_t)generic_fft_len(h) * sizeof(double2);
            GStftArgs<T> sa{};
            sa.gg = gg; sa.tb = gt; sa.x = gin; sa.X = gX;
            { auto kern_ = gk_stft<T, true>;
              B200_LAUNCH(kern_, dim3((unsigned)g.T, (unsigned)nu), dim3(thr_fft), smem_fft, st, sa); }
            GIstftArgs ia{};
            ia.gg = gg; ia.tb = gt; ia.X = gX; ia.M = (const double*)(store + (size_t)u0 * kp.unit_bytes); ia.frames = gFr;
            ia.dbg_ul = -1;
            B200_LAUNCH(gk_istft, dim3((unsigned)g.T, (unsigned)nu), dim3(thr_fft), smem_fft, st, ia);
            GOlaArgs<T> oa{};
            oa.gg = gg; oa.tb = gt; oa.frames = gFr; oa.adj = adj; oa.adj_pitch = adj_pitch;
            { auto kern_ = gk_ola<T, true>;
              B200_LAUNCH(kern_, dim3((unsigned)grid_1d(g.Lp, 256, 1 << 16), (unsigned)nu), dim3(256), 0, st, oa); }
        } else {
            float* adj = (float*)(ws + off_adj);
            CK(h, cudaMemsetAsync(adj, 0, (size_t)nu * adj_pitch * adj_es, st));   // hops no frame of the centre reaches
            K2Args a2{};
            a2.g = g; a2.tb = tb; a2.x = gin; a2.y = nullptr; a2.zcache = nullptr; a2.nt = nt; a2.dbg.ul = -1;
            a2.adj = adj; a2.adj_pitch = adj_pitch;
            if (stat) {
                unsigned short* num = (unsigned short*)ws;
                SmoothArgs sa{};
                sa.n_units = nu; sa.T = g.T; sa.nf = nf; sa.nt = nt; sa.tf_lo = tf_lo; sa.tf_hi = tf_hi; sa.TT = 32;
                sa.bits = (const unsigned*)(store + (size_t)u0 * kp.unit_bytes);
                sa.rowflag = (const unsigned*)(store + kp.off_rowflag + (size_t)u0 * kFW * 4);
                sa.num = num;
                launch_stationary_numerators(h, sa, st);
                a2.num = num;
                a2.pD = (float)(p.prop_decrease / D);
                a2.one_minus_p = (float)(1.0 - p.prop_decrease);
            } else {
                a2.fmask = (const float*)(store + (size_t)u0 * kp.unit_bytes);
            }
            // output hops: every hop the frames [h_lo - 3, h_hi - 1] overlap (k2_synthesize<.., ADJ>)
            const int NH = NFFT / g.H;
            const long long hops = (std::min(h_hi - 1, g.T - 1) + NH) - std::max(0, h_lo - (NH - 1));
            const int res_k2 = two_k ? h->num_sm * 2 : resident;
            long long run = ((long long)nu * hops + (long long)res_k2 * kWarps * 4 - 1) / ((long long)res_k2 * kWarps * 4);
            run = std::max(16LL, std::min(128LL, run));
            run += run & 1;
            a2.run = (int)run;
            a2.n_runs = (int)((hops + a2.run - 1) / a2.run);
            const dim3 grid2(grid_1d((long long)nu * a2.n_runs, kWarps, res_k2));
            if (two_k) {
                K22Args a22{};
                a22.g = g; a22.x = (const float*)gk; a22.y = nullptr; a22.fmask = a2.fmask; a22.dbg.ul = -1;
                a22.tb.wa2 = h->d_wa2; a22.tb.ws2 = h->d_ws2; a22.tb.tw = h->d_tw; a22.tb.w2k = h->d_w2k;
                a22.tb.invn2 = h->d_invn2; a22.tb.ws_to_w = h->ws_to_w;
                a22.run = a2.run; a22.n_runs = a2.n_runs; a22.adj = adj; a22.adj_pitch = adj_pitch;
                B200_LAUNCH(k2_synthesize_2k<true>, grid2, dim3(kThreads), k22_smem_floats() * 4, st, a22);
            } else if (stat) {
                auto kern2 = k2_synthesize<8, false, T, true>;
                B200_LAUNCH(kern2, grid2, dim3(kThreads), k2_smem_floats(g.H) * 4, st, a2);
            } else {
                auto kern2 = k2_synthesize<8, true, T, true>;
                B200_LAUNCH(kern2, grid2, dim3(kThreads), k2_smem_floats(g.H) * 4, st, a2);
            }
        }
        // the ordered sum of this batch's spans into grad
        const long long cf = g.u0 / C, cl = (g.u0 + nu - 1) / C;
        const long long s_lo = std::max(0LL, cf * g.step - g.pad), s_hi = std::min<long long>(N, (cl + 1) * g.step + g.pad);
        // (channels ride on gridDim.y, at most 65535 per launch)
        for (long long c0 = 0; s_hi > s_lo && c0 < C; c0 += 65535) {
            const long long nc = std::min(C - c0, 65535LL);
            const dim3 grid3(grid_1d(s_hi - s_lo, 256, std::max(1, 8192 / (int)std::min<long long>(nc, 8192))), (unsigned)nc);
            if (generic) {
                auto kern3 = k_adj_gather<double, T>;
                B200_LAUNCH(kern3, grid3, dim3(256), 0, st, (const double*)(ws + off_adj), adj_pitch, grad,
                            (long long)grad_stride, g, s_lo, s_hi, (int)c0);
            } else {
                auto kern3 = k_adj_gather<float, T>;
                B200_LAUNCH(kern3, grid3, dim3(256), 0, st, (const float*)(ws + off_adj), adj_pitch, grad,
                            (long long)grad_stride, g, s_lo, s_hi, (int)c0);
            }
        }
        CK(h, cudaGetLastError());
    }
    return B200GATE_OK;
}
}  // namespace

extern "C" {

int b200gate_adjoint(b200gate_handle* h, const void* store, const void* g_in, void* grad, int dtype, int64_t C, int64_t N,
                     int64_t g_stride, int64_t grad_stride, int is_device, void* stream) {
    if (!h) return B200GATE_ERR_ARG;
    MaskPlan kp{};
    int rc = mask_plan(h, C, N, &kp);
    if (rc) return rc;
    if (!store || !g_in || !grad || (dtype != B200GATE_F32 && dtype != B200GATE_F64))
        return fail(h, B200GATE_ERR_ARG, "b200gate_adjoint: null pointer, or a gradient dtype other than float32 / float64");
    if (!is_device) return fail(h, B200GATE_ERR_ARG, "b200gate_adjoint takes device pointers");
    if (h->s_open) return fail(h, B200GATE_ERR_STATE, "a stream is open on this handle (b200gate_stream_finish first)");
    // the centre the forward wrote, [o_lo, o_hi): g is read there only, so a virtual base over a shorter slab will do
    const long long o_lo = (kp.Ubase / C) * kp.g.step;
    const long long o_hi = std::min<long long>(N, (kp.Ubase + kp.U) / C * kp.g.step);
    if (grad_stride < N || (C > 1 && g_stride < (h->range_mode == 0 ? N : o_hi - o_lo)))
        return fail(h, B200GATE_ERR_ARG, "row strides too small");
    const MaskPlan* mp = &kp;
    bool found = false;
    for (const auto& r : h->kept)
        if (r.store == store) {
            found = r.C == C && r.N == N && r.mode == h->range_mode && r.bytes == mp->bytes &&
                    (r.mode == 0 || (r.a == h->range_a && (r.mode == 2 || r.b == h->range_b)));
            break;
        }
    if (!found)
        return fail(h, B200GATE_ERR_STATE, "the mask store holds no masks of a b200gate_run of this handle with C = %lld, "
                    "N = %lld and the current range", (long long)C, (long long)N);
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == B200GATE_F64)
        return adjoint_impl<double>(h, kp, (const char*)store, (const double*)g_in, (double*)grad, g_stride, grad_stride, st);
    return adjoint_impl<float>(h, kp, (const char*)store, (const float*)g_in, (float*)grad, g_stride, grad_stride, st);
}

// ---- streaming: the recording arrives in blocks (include/b200gate.h) --------------------------------------------------
namespace {

// samples returned once R have been received: every chunk whose padded span [i cs - pad, (i + 1) cs + pad) has arrived,
// and nothing while the recording could still turn out to be one padded chunk (N <= chunk_size, base.py:222)
long long stream_emitted(const b200gate_params& p, long long R) {
    const long long cs = p.chunk_size;
    return R > cs ? cs * std::max(0LL, (R - p.padding) / cs) : 0;
}

// A pinned staging buffer of at least `bytes` (host pushes of pageable memory), from the process-wide pool.
int stream_pinned(b200gate_handle* h, void** buf, size_t* have, size_t bytes) {
    if (*have >= bytes) return B200GATE_OK;
    g_pinned_pool.give(*buf, *have);
    *buf = g_pinned_pool.take(bytes, have);
    if (!*buf) { *have = 0; return fail(h, B200GATE_ERR_NOMEM, "pinned staging buffer (%zu bytes)", bytes); }
    return B200GATE_OK;
}

// Run chunks [E / cs, E_new / cs) (or, last == true, everything from E to the end of a recording of R samples) from the
// window, write them to out + (E - first_col) columns, and advance E.  One run_core call: the batching of an offline run.
int stream_emit(b200gate_handle* h, long long E_new, bool last, void* out, long long out_stride, long long first_col,
                int is_device, cudaStream_t st) {
    const b200gate_params& p = h->p;
    const long long R = h->s_R, E = h->s_E, C = h->s_C;
    const size_t es = dtype_size(h->s_dtype);
    if (E_new <= E) return B200GATE_OK;
    const bool stage = !is_device && !host_pointer_is_pinned(out);
    int rc;
    if (!is_device && (rc = ensure(h, &h->d_sout, &h->sout_bytes, (size_t)C * h->s_ocap * es))) return rc;
    if (stage && (rc = stream_pinned(h, &h->hp_out[0], &h->hp_out_bytes[0], (size_t)C * h->s_ocap * es))) return rc;
    const void* xv = (const char*)h->d_swin - (size_t)h->s_lo * es;
    // host callers: the library's output buffer (pitch s_ocap, column 0 = sample E), then one copy out
    void* yv = is_device ? (char*)out - (size_t)first_col * es : (char*)h->d_sout - (size_t)E * es;
    const long long ys = is_device ? out_stride : h->s_ocap;
    const int32_t mode0 = h->range_mode;
    const long long a0 = h->range_a, b0 = h->range_b;
    if (last && R <= p.chunk_size) h->range_mode = 0;          // one padded chunk: the whole recording
    else { h->range_mode = 1; h->range_a = E / p.chunk_size; h->range_b = (E_new - 1) / p.chunk_size; }
    rc = run_core(h, xv, yv, h->s_dtype, C, R, h->s_cap, ys, 1, st, h->s_lo);
    h->range_mode = mode0; h->range_a = a0; h->range_b = b0;
    if (rc) return rc;
    if (!is_device) {
        const long long m = E_new - E;
        void* dst = (char*)out + (size_t)(E - first_col) * es;
        CK(h, cudaMemcpy2DAsync(stage ? h->hp_out[0] : dst, stage ? (size_t)m * es : (size_t)out_stride * es, h->d_sout,
                                (size_t)h->s_ocap * es, (size_t)m * es, (size_t)C, cudaMemcpyDeviceToHost, st));
        CK(h, cudaStreamSynchronize(st));
        if (stage) parallel_rows_copy(dst, (size_t)out_stride * es, h->hp_out[0], (size_t)m * es, (size_t)m * es, (size_t)C,
                                      h->host_threads);
    }
    h->s_E = E_new;
    return B200GATE_OK;
}

// a stationary numpy-surface stream needs thresholds before it returns a chunk; the torch surfaces can always take each
// unit's own statistics
bool stream_needs_thresholds(const b200gate_handle* h) {
    return h->p.stationary && h->p.surface == B200GATE_SURFACE_NUMPY && !h->have_thresh;
}

int stream_check_space(b200gate_handle* h, int is_device) {
    if (h->ts_open) return fail(h, B200GATE_ERR_STATE, kTsOpen);
    if (!h->s_open) return fail(h, B200GATE_ERR_STATE, "no open stream (b200gate_stream_begin first)");
    if (h->s_is_device >= 0 && h->s_is_device != (is_device ? 1 : 0))
        return fail(h, B200GATE_ERR_ARG, "every push of a stream must use the same memory space (is_device)");
    return B200GATE_OK;
}

}  // namespace

int b200gate_stream_begin(b200gate_handle* h, int dtype, int64_t C) {
    if (!h) return B200GATE_ERR_ARG;
    if (h->ts_open) return fail(h, B200GATE_ERR_STATE, kTsOpen);
    h->s_open = false;
    if (h->p.surface == B200GATE_SURFACE_TORCH)
        return fail(h, B200GATE_ERR_ARG, "streaming needs the numpy or the chunked torch surface");
    if (h->p.chunk_size <= 0)
        return fail(h, B200GATE_ERR_ARG, "streaming needs chunk_size > 0 (without chunks nothing can be returned early)");
    const size_t es = dtype_size(dtype);
    if (es == 0 || C <= 0) return fail(h, B200GATE_ERR_ARG, "bad argument");
    const long long cs = h->p.chunk_size, pad = h->p.padding;
    // window alignment: its first sample sits at an absolute index whose byte offset is a multiple of 16, and so does
    // its row pitch, so the kernels see the addresses of an offline run of an aligned recording
    const long long A = 16 / (long long)es;
    // a push is consumed in slices of whole chunks, ~256 MB of input each (the slab size of the offline host path)
    long long per = 256LL << 20;
    if (const char* e = getenv("B200GATE_SLAB_MB")) per = std::max(1LL, atoll(e)) << 20;
    long long k = std::max(1LL, std::min(64LL, per / std::max(1LL, C * cs * (long long)es)));
    if (const char* e = getenv("B200GATE_STREAM_SLICE_CHUNKS")) k = std::max(1LL, atoll(e));   // tests / tuning
    const long long S = k * cs;
    // retained before a slice: [align(E - pad), R) with R - E < cs + pad, i.e. fewer than Lmax samples.  With a pitch of
    // S + 2 Lmax the window is compacted only when the move's source and destination do not overlap.
    const long long Lmax = 2 * pad + cs + A;
    h->s_slice = S;
    h->s_cap = (S + 2 * Lmax + A - 1) / A * A;
    h->s_ocap = (S + cs + pad + A - 1) / A * A;                // a slice returns < S + cs samples, the end < cs + pad
    int rc;
    if ((rc = ensure(h, &h->d_swin, &h->swin_bytes, (size_t)C * h->s_cap * es))) return rc;
    h->s_dtype = dtype; h->s_C = C; h->s_R = 0; h->s_E = 0; h->s_lo = 0; h->s_is_device = -1;
    h->s_open = true;
    return B200GATE_OK;
}

int b200gate_stream_push(b200gate_handle* h, const void* in, int64_t n, int64_t in_stride, int is_device, void* out,
                         int64_t out_stride, int64_t out_capacity, int64_t* n_out, void* stream) {
    if (!h) return B200GATE_ERR_ARG;
    int rc;
    if ((rc = stream_check_space(h, is_device))) return rc;
    const b200gate_params& p = h->p;
    const long long C = h->s_C;
    if (!n_out || n < 0 || (n > 0 && (!in || in_stride < n)) || !out || out_stride < out_capacity)
        return fail(h, B200GATE_ERR_ARG, "bad argument");
    if (out_capacity < n + p.chunk_size)
        return fail(h, B200GATE_ERR_ARG, "out_capacity %lld < n + chunk_size = %lld", (long long)out_capacity,
                    (long long)(n + p.chunk_size));
    const long long E0 = h->s_E, E_end = stream_emitted(p, h->s_R + n);
    if (E_end > E0 && stream_needs_thresholds(h))
        return fail(h, B200GATE_ERR_STATE, "stationary stream: set the noise thresholds before the first chunk is returned");
    *n_out = E_end - E0;
    if (n == 0) return B200GATE_OK;
    h->s_is_device = is_device ? 1 : 0;
    cudaStream_t st = (cudaStream_t)stream;
    const size_t es = dtype_size(h->s_dtype);
    const long long S = h->s_slice, A = 16 / (long long)es;
    const bool stage_in = !is_device && !host_pointer_is_pinned(in);
    if (stage_in && (rc = stream_pinned(h, &h->hp_in[0], &h->hp_in_bytes[0], (size_t)C * S * es))) return rc;
    for (long long off = 0; off < n;) {
        const long long s = std::min(S, n - off);
        if (h->s_R - h->s_lo + s > h->s_cap) {                 // compact: keep [align(E - pad), R)
            const long long lo = std::max(0LL, h->s_E - p.padding) / A * A, L = h->s_R - lo;
            if (L > 0)
                CK(h, cudaMemcpy2DAsync(h->d_swin, (size_t)h->s_cap * es, (char*)h->d_swin + (size_t)(lo - h->s_lo) * es,
                                        (size_t)h->s_cap * es, (size_t)L * es, (size_t)C, cudaMemcpyDeviceToDevice, st));
            h->s_lo = lo;
        }
        // the slice's samples cross to the device once, behind the retained ones
        void* dst = (char*)h->d_swin + (size_t)(h->s_R - h->s_lo) * es;
        const void* src = (const char*)in + (size_t)off * es;
        size_t spitch = (size_t)in_stride * es;
        if (stage_in) {
            CK(h, cudaStreamSynchronize(st));                   // the previous slice has left the staging buffer
            parallel_rows_copy(h->hp_in[0], (size_t)s * es, src, spitch, (size_t)s * es, (size_t)C, h->host_threads);
            src = h->hp_in[0];
            spitch = (size_t)s * es;
        }
        CK(h, cudaMemcpy2DAsync(dst, (size_t)h->s_cap * es, src, spitch, (size_t)s * es, (size_t)C,
                                is_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, st));
        h->s_R += s;
        off += s;
        if ((rc = stream_emit(h, stream_emitted(p, h->s_R), false, out, out_stride, E0, is_device, st))) {
            h->s_open = false;
            return rc;
        }
    }
    if (!is_device) CK(h, cudaStreamSynchronize(st));
    return B200GATE_OK;
}

int b200gate_stream_finish(b200gate_handle* h, void* out, int64_t out_stride, int64_t out_capacity, int64_t* n_out,
                           void* stream) {
    if (!h) return B200GATE_ERR_ARG;
    int rc;
    if ((rc = stream_check_space(h, h->s_is_device > 0))) return rc;
    const b200gate_params& p = h->p;
    if (!n_out || !out || out_stride < out_capacity) return fail(h, B200GATE_ERR_ARG, "bad argument");
    if (out_capacity < p.chunk_size + p.padding)
        return fail(h, B200GATE_ERR_ARG, "out_capacity %lld < chunk_size + padding = %lld", (long long)out_capacity,
                    (long long)(p.chunk_size + p.padding));
    const long long E0 = h->s_E, R = h->s_R;
    if (R > E0 && stream_needs_thresholds(h))
        return fail(h, B200GATE_ERR_STATE, "stationary stream: set the noise thresholds before the first chunk is returned");
    rc = stream_emit(h, R, true, out, out_stride, E0, h->s_is_device > 0, (cudaStream_t)stream);
    h->s_open = false;
    if (rc) return rc;
    *n_out = R - E0;
    // chunked torch surface: a recording of one padded chunk returns what its torch output holds past the padding
    if (p.surface == B200GATE_SURFACE_TORCH_CHUNKED && R <= p.chunk_size) {
        const long long Lp = R + 2 * p.padding;
        *n_out = std::min<long long>(R, (Lp / p.hop_length) * p.hop_length + (p.n_fft & 1) - p.padding);
    }
    return B200GATE_OK;
}


// ---- TorchGate.stream(): the non-stationary TorchGate on rows that arrive block by block ------------------------------
// Every stage of the gate looks ahead a bounded number of frames: frame t of torch.stft(center=True) needs samples up to
// t H + n_fft / 2, the moving mean of frame t needs |X| up to frame t + right, the smoothing of frame t masks up to t + nt,
// and the overlap-add of hop h frames h - 3 .. h.  So after R samples per row the stream can finish
//   nA(R) = 2 floor(c / 2) frames of analysis, c = floor((R - n_fft / 2) / H) + 1 (the frames whose samples are in),
//   nM = nA - 1 - right frames of moving mean, nS = nM - nt frames of smoothing,
//   hops [2, hb), hb = 2 floor(nS / 2): output samples [0, (hb - 2) H)
// (each clamped at 0).  Frames are analysed and synthesised in the global pairs (2j, 2j+1) of b200gate_run, the moving
// mean carries its double running sum per (row, bin), and the smoothing restarts in every frame, so every returned sample
// equals b200gate_run on the whole rows in every bit; b200gate_tstream_finish does the last frames with T = R / H + 1.
namespace {

long long ts_hops_done(const b200gate_handle* h, long long R) {      // hb(R) above
    const int n = h->p.n_movemean, right = n - 1 - (n - 1) / 2;
    if (R < kN / 2) return 2;
    const long long c = (R - kN / 2) / h->p.hop_length + 1;
    const long long nS = (c & ~1LL) - 1 - right - h->p.n_grad_time;
    return std::max(2LL, nS & ~1LL);
}

// One row's stage targets after R received samples (T = 0) or at its end (T = R / H + 1 frames), from the moving mean
// and smoothing done so far (nM0, nS0) and the first hop not yet returned (ha0): analysis to nA, moving mean to nM,
// smoothing to nS, synthesis to hop hb.
struct TsTarget { long long nA, nM, nS, hb; };
TsTarget ts_target(const b200gate_handle* h, long long R, long long T, long long nM0, long long nS0, long long ha0) {
    if (T > 0) return {T, T, T, T + 1};
    const int n = h->p.n_movemean, right = n - 1 - (n - 1) / 2;
    const long long c = R >= kN / 2 ? (R - kN / 2) / h->p.hop_length + 1 : 0;
    const long long nA = c & ~1LL, nM = std::max(nM0, nA - 1 - right), nS = std::max(nS0, nM - h->p.n_grad_time);
    return {nA, nM, nS, std::max(ha0, nS & ~1LL)};
}

// The launches of one slice: frames [a0, a1) of analysis, [m0, m1) of moving mean, [s0, s1) of smoothing and hops
// [ha, hb) of synthesis, under the frame bound Tb (INT_MAX while the end is unknown), R samples in the window x (the
// virtual base of sample 0), hop ha's first sample to out[b][0].  SESS: every row's ranges, bound, window start and
// output offset come from the device table `rows`; the ranges here start at 0 and end at the largest span of any row,
// which sizes the grids (rows with less to do leave early), and Tb, R and x are unused.
struct TsSlice { long long a0, a1, m0, m1, s0, s1, ha, hb; int Tb; long long R; const float* x; };

extern "C++" {                                             // (this file's entry points have C linkage)
template <bool SESS>
int ts_launch(b200gate_handle* h, const TsSlice& s, const SessRow* rows, float* out, long long out_stride, cudaStream_t st) {
    const b200gate_params& p = h->p;
    const int H = p.hop_length, nt = p.n_grad_time, nf = p.n_grad_freq, ring = h->ts_ring;
    const int n = p.n_movemean;
    const int B = (int)h->ts_B;
    const Tables tb = device_tables(h);
    StreamWin sw{};
    sw.ring = ring;
    if (s.a1 > s.a0) {
        K1nArgs a1{};
        a1.g.H = H; a1.g.C = B; a1.g.T = (int)s.a1; a1.g.n_chunks = 1; a1.g.n_total = s.R; a1.g.step = s.R; a1.g.pad = 0;
        a1.g.Lp = s.R; a1.g.in_stride = h->ts_cap; a1.g.u0 = 0; a1.g.n_units = B;
        a1.tb = tb; a1.x = SESS ? h->d_ts_win : s.x; a1.mag = h->d_ts_mag; a1.dbg.ul = -1; a1.zcache = h->d_ts_z;
        a1.zpairs = ring / 2; a1.z_lo = 0; a1.z_hi = INT_MAX;
        sw.f0 = (int)s.a0;
        a1.sw = sw; a1.rows = rows;
        a1.run = 2;                                           // one frame pair per work item (pairs are global either way)
        a1.n_runs = (int)((s.a1 - s.a0 + 1) / 2);
        auto kern_ = k1n_magnitude<8, float, false, true, SESS>;
        B200_LAUNCH(kern_, dim3(grid_1d((long long)B * a1.n_runs, kWarps, h->num_sm * 3)), dim3(kThreads),
                    k1n_smem_floats() * 4, st, a1);
    }
    if (s.m1 > s.m0) {
        TMovArgs ma{};
        ma.n_units = B; ma.T = s.Tb; ma.n_movemean = n; ma.n_thresh = (float)p.thresh_n_mult;
        ma.inv_temp = (float)p.sigmoid_slope; ma.p = (float)p.prop_decrease; ma.mag = h->d_ts_mag; ma.m0 = h->d_ts_m0;
        sw.f0 = (int)s.m0;
        ma.sw = sw; ma.f1 = (int)s.m1; ma.run = h->d_ts_run; ma.rows = rows;
        auto kern_ = k_tgate_movmean<false, true, SESS>;
        B200_LAUNCH(kern_, dim3(grid_1d((long long)B * kFPad, 128, 1 << 30)), dim3(128), 0, st, ma);
    }
    if (s.s1 > s.s0) {
        SmoothFArgs sa{};
        sa.n_units = B; sa.T = s.Tb; sa.nf = nf; sa.nt = nt; sa.tf_lo = (int)s.s0; sa.tf_hi = (int)s.s1; sa.F = kF; sa.FPad = kFPad;
        sa.p = 1.0f; sa.one_minus_p = 0.0f;                  // (the torch surface blends in k_tgate_movmean)
        sa.m0 = h->d_ts_m0; sa.m2 = h->d_ts_mask; sa.sw = sw; sa.rows = rows;
        launch_smooth_float<false, true, SESS>(sa, nf, nt, (int)s.s0, (int)s.s1, B, 0, st);   // (extents checked at begin)
    }
    if (s.hb > s.ha) {
        // hops [ha, hb): Geom's padded-chunk view with pad = (ha - 2) H puts the first of them at h_lo and output sample
        // (ha - 2) H at out[b][0]; while the end is unknown, T = hb + 1 keeps every hop interior
        const long long P = (s.ha - 2) * H;
        const long long out_len = (s.hb - 2) * H - P;
        K2Args a2{};
        a2.g.H = H; a2.g.C = B; a2.g.T = (int)std::min<long long>(s.Tb, s.hb + 1); a2.g.n_chunks = 1; a2.g.n_total = out_len;
        a2.g.step = out_len; a2.g.pad = P; a2.g.Lp = out_len + P; a2.g.out_stride = out_stride; a2.g.u0 = 0; a2.g.n_units = B;
        a2.tb = tb; a2.y = out; a2.fmask = h->d_ts_mask; a2.zcache = h->d_ts_z; a2.zpairs = ring / 2; a2.nt = nt;
        a2.dbg.ul = -1; a2.sw = sw; a2.rows = rows;
        const long long hops = s.hb - s.ha;
        long long want = (long long)h->num_sm * 3 * kWarps * 4;
        long long run = std::max(16LL, std::min(128LL, ((long long)B * hops + want - 1) / want));
        run += run & 1;                                       // work items end on odd frames, as in b200gate_run
        a2.run = (int)run;
        a2.n_runs = (int)((hops + run - 1) / run);
        auto kern_ = k2c_synthesize<8, kMaskF32, float, false, true, SESS>;
        B200_LAUNCH(kern_, dim3(grid_1d((long long)B * a2.n_runs, kWarps, h->num_sm * 3)), dim3(kThreads),
                    k2c_smem_bytes<kMaskF32>(), st, a2);
    }
    CK(h, cudaGetLastError());
    return B200GATE_OK;
}
}  // extern "C++"

// Advance the lockstep stream to R = h->ts_R received samples (T = 0) or to its end (T = R / H + 1 frames): analysis,
// moving mean, smoothing, synthesis of what has become final.  The hops returned go to out[b][0, ...) (row stride
// out_stride).
int ts_advance(b200gate_handle* h, long long T, float* out, long long out_stride, cudaStream_t st) {
    const TsTarget t = ts_target(h, h->ts_R, T, h->ts_nM, h->ts_nS, h->ts_ha);
    const TsSlice s{h->ts_nA, t.nA, h->ts_nM, t.nM, h->ts_nS, t.nS, h->ts_ha, t.hb, T > 0 ? (int)T : INT_MAX, h->ts_R,
                    h->d_ts_win - h->ts_lo};
    const int rc = ts_launch<false>(h, s, nullptr, out, out_stride, st);
    if (rc) return rc;
    h->ts_nA = t.nA; h->ts_nM = t.nM; h->ts_nS = t.nS; h->ts_ha = t.hb;
    return B200GATE_OK;
}

void ts_release(b200gate_handle* h) {
    if (h->d_ts) cudaFree(h->d_ts);
    h->d_ts = nullptr;
    h->ts_open = false;
    h->ts_mode = 0;
}

const char* const kTsLockstep = "this torch stream advances its rows together (b200gate_tstream_push / _finish)";
const char* const kTsPerRow = "this torch stream advances its rows one by one (b200gate_tstream_push_rows / _end_rows / _reset_rows)";

// The per-row calls: an open stream that has not taken the lockstep calls.
int sess_check(b200gate_handle* h) {
    if (!h->ts_open) return fail(h, B200GATE_ERR_STATE, "no open torch stream (b200gate_tstream_begin first)");
    if (h->ts_mode == 1) return fail(h, B200GATE_ERR_STATE, kTsLockstep);
    return B200GATE_OK;
}

// rows[0, k): in range and none twice
int sess_check_rows(b200gate_handle* h, const int64_t* rows, int64_t k) {
    if (k < 0 || (k > 0 && !rows)) return fail(h, B200GATE_ERR_ARG, "bad argument");
    std::vector<char> seen((size_t)h->ts_B, 0);
    for (int64_t i = 0; i < k; ++i) {
        if (rows[i] < 0 || rows[i] >= h->ts_B)
            return fail(h, B200GATE_ERR_ARG, "row %lld out of range [0, %lld)", (long long)rows[i], h->ts_B);
        if (seen[(size_t)rows[i]]++) return fail(h, B200GATE_ERR_ARG, "row %lld listed twice", (long long)rows[i]);
    }
    return B200GATE_OK;
}

// Row r's table entry for a slice that brings it to r.R samples (T = 0) or ends it (T = R / H + 1); its output sample j
// goes to out[y + j].  Advances r and widens the largest spans in `span`.
void sess_fill(const b200gate_handle* h, b200gate_handle::TsRow& r, SessRow& e, long long T, long long y, TsSlice& span) {
    const TsTarget t = ts_target(h, r.R, T, r.nM, r.nS, r.ha);
    e.R = r.R; e.lo = r.lo; e.y = y; e.T = T > 0 ? (int)T : INT_MAX;
    e.a0 = (int)r.nA; e.a1 = (int)t.nA; e.m0 = (int)r.nM; e.m1 = (int)t.nM;
    e.s0 = (int)r.nS; e.s1 = (int)t.nS; e.ha = (int)r.ha; e.hb = (int)t.hb;
    span.a1 = std::max(span.a1, t.nA - r.nA); span.m1 = std::max(span.m1, t.nM - r.nM);
    span.s1 = std::max(span.s1, t.nS - r.nS); span.hb = std::max(span.hb, t.hb - r.ha);
    r.nA = t.nA; r.nM = t.nM; r.nS = t.nS; r.ha = t.hb;
}

// The next slot of the upload ring; waits for that slot's previous copy to have left it (the only wait of the per-row
// calls: it happens when the host is kSessSlots slices ahead of the device).
SessRow* sess_slot(b200gate_handle* h, int* k) {
    *k = (int)(h->sess_slices++ % kSessSlots);
    cudaEventSynchronize(h->ev_sess[*k]);
    SessRow* tab = h->hp_sess + (size_t)*k * h->ts_B;
    memset(tab, 0, (size_t)h->ts_B * sizeof(SessRow));
    for (long long b = 0; b < h->ts_B; ++b) { tab[b].ha = tab[b].hb = 2; tab[b].T = INT_MAX; }   // (nothing to do)
    return tab;
}

// Upload slot k's table and enqueue its slice: the copy-in of block columns [off, off + S) (in != nullptr), then the
// four stages.
int sess_submit(b200gate_handle* h, int k, const TsSlice& span, const float* in, long long in_stride, long long off,
                float* out, cudaStream_t st) {
    const long long B = h->ts_B;
    SessRow* d_tab = h->d_sess + (size_t)k * B;
    CK(h, cudaMemcpyAsync(d_tab, h->hp_sess + (size_t)k * B, (size_t)B * sizeof(SessRow), cudaMemcpyHostToDevice, st));
    CK(h, cudaEventRecord(h->ev_sess[k], st));
    if (in) {
        SessCopyArgs ca{in, in_stride, off, h->d_ts_win, h->ts_cap, d_tab};
        B200_LAUNCH(k_sess_copy_in, dim3((unsigned)B), dim3(256), 0, st, ca);
    }
    return ts_launch<true>(h, span, d_tab, out, 0, st);
}

}  // namespace

int b200gate_tstream_begin(b200gate_handle* h, int64_t n_rows) {
    if (!h) return B200GATE_ERR_ARG;
    const b200gate_params& p = h->p;
    if (p.surface != B200GATE_SURFACE_TORCH || p.stationary || h->generic || p.n_fft != kN || p.win_length != kN ||
        p.hop_length != 256)
        return fail(h, B200GATE_ERR_STATE, "torch streams need a non-stationary TORCH-surface handle at n_fft = win_length "
                    "= 1024, hop_length = 256 (the stationary gate's statistics span the whole row)");
    if (h->s_open) return fail(h, B200GATE_ERR_STATE, "a stream is open on this handle (b200gate_stream_finish first)");
    if (n_rows <= 0 || n_rows > 0x7fffffffLL / kFPad) return fail(h, B200GATE_ERR_ARG, "bad argument");
    const int nf = p.n_grad_freq, nt = p.n_grad_time;
    const bool box = nf >= 1 && nf <= 12 && smoothb_smem_bytes(kFPad, nt) <= 200 * 1024;
    if (!box && smooths_smem_bytes(kFPad, nf, nt) > 200 * 1024)
        return fail(h, B200GATE_ERR_ARG, "smoothing extents (%d, %d) beyond the shared-memory ring of the streaming smoothing",
                    nf, nt);
    ts_release(h);
    const int n = p.n_movemean, left = (n - 1) / 2, right = n - 1 - left;
    // A push is consumed in slices of S samples: a slice adds at most S / H + 2 frames to each stage.  Frames live in the
    // rings from their analysis until the last stage reads them: the moving mean reads |X| from nM - left to nA, the
    // smoothing masks from nS - nt to nM, the synthesis spectra and masks from hop ha - 4 (<= nS - 5) on.  Between
    // slices nA - nM <= right + 1 and nM - nS <= nt, so left + right + 2 nt + S / H + 8 frames always suffice.
    const long long S = 4096;
    long long need = left + right + 2LL * nt + S / 256 + 16, ring = 16;
    while (ring < need) ring *= 2;
    if (ring > (1 << 20)) return fail(h, B200GATE_ERR_ARG, "n_movemean %d: frame rings too large", n);
    // the sample window keeps [nA H - n_fft / 2, R) (< 2 H + n_fft samples) before a slice; with a pitch of
    // S + 2 (2 H + n_fft) a compaction never moves a span onto itself
    const long long cap = S + 2 * (2 * 256 + kN);
    const size_t B = (size_t)n_rows;
    auto al = [](size_t v) { return (v + 255) / 256 * 256; };
    const size_t o_win = 0, o_z = o_win + al(B * cap * 4), o_mag = o_z + al(B * (size_t)(ring / 2) * 1024 * 8);
    const size_t o_m0 = o_mag + al(B * ring * kFPad * 4), o_mask = o_m0 + al(B * ring * kFPad * 4);
    const size_t o_run = o_mask + al(B * ring * kFPad * 4), o_sess = o_run + al(B * kFPad * 8);
    const size_t sess_bytes = (size_t)kSessSlots * B * sizeof(SessRow), bytes = o_sess + al(sess_bytes);
    if (h->ev_sess.empty()) {
        h->ev_sess.assign(kSessSlots, nullptr);
        for (cudaEvent_t& ev : h->ev_sess) CK(h, cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    }
    if (h->hp_sess_bytes < sess_bytes) {
        g_pinned_pool.give(h->hp_sess, h->hp_sess_bytes);
        h->hp_sess = (SessRow*)g_pinned_pool.take(sess_bytes, &h->hp_sess_bytes);
        if (!h->hp_sess) { h->hp_sess_bytes = 0; return fail(h, B200GATE_ERR_NOMEM, "pinned row tables (%zu bytes)", sess_bytes); }
    }
    cudaError_t e = cudaMalloc(&h->d_ts, bytes);
    if (e != cudaSuccess) {
        cudaGetLastError();
        h->d_ts = nullptr;
        return fail(h, B200GATE_ERR_NOMEM, "cudaMalloc(%zu bytes) for the torch stream failed: %s", bytes, cudaGetErrorString(e));
    }
    char* base = (char*)h->d_ts;
    h->d_ts_win = (float*)(base + o_win); h->d_ts_z = (float2*)(base + o_z); h->d_ts_mag = (float*)(base + o_mag);
    h->d_ts_m0 = (float*)(base + o_m0); h->d_ts_mask = (float*)(base + o_mask); h->d_ts_run = (double*)(base + o_run);
    h->d_sess = (SessRow*)(base + o_sess);
    h->ts_row.assign(B, b200gate_handle::TsRow{});
    h->ts_y0.assign(B, 0);
    h->ts_B = n_rows; h->ts_R = 0; h->ts_lo = 0; h->ts_cap = cap; h->ts_slice = S; h->ts_ring = (int)ring;
    h->ts_nA = 0; h->ts_nM = 0; h->ts_nS = 0; h->ts_ha = 2;
    h->ts_open = true;
    return B200GATE_OK;
}

int b200gate_tstream_push(b200gate_handle* h, const float* in, int64_t n, int64_t in_stride, float* out, int64_t out_stride,
                          int64_t out_capacity, int64_t* n_out, void* stream) {
    if (!h) return B200GATE_ERR_ARG;
    if (!h->ts_open) return fail(h, B200GATE_ERR_STATE, "no open torch stream (b200gate_tstream_begin first)");
    if (!n_out || n < 0 || (n > 0 && (!in || in_stride < n)) || out_capacity < 0 || (out_capacity > 0 && !out) ||
        (h->ts_B > 1 && out_stride < out_capacity))
        return fail(h, B200GATE_ERR_ARG, "bad argument");
    if (h->ts_mode == 2) return fail(h, B200GATE_ERR_STATE, kTsPerRow);
    const long long H = h->p.hop_length;
    const long long m = (ts_hops_done(h, h->ts_R + n) - h->ts_ha) * H;
    if (out_capacity < m)
        return fail(h, B200GATE_ERR_ARG, "out_capacity %lld < %lld samples returned by this push", (long long)out_capacity, m);
    *n_out = m;
    h->ts_mode = 1;
    if (n == 0) return B200GATE_OK;
    cudaStream_t st = (cudaStream_t)stream;
    const long long B = h->ts_B, S = h->ts_slice, ha0 = h->ts_ha;
    int rc;
    for (long long off = 0; off < n;) {
        const long long s = std::min(S, n - off);
        if (h->ts_R - h->ts_lo + s > h->ts_cap) {            // compact: keep the samples of frames nA on
            const long long lo = std::max(0LL, h->ts_nA * H - kN / 2), L = h->ts_R - lo;
            if (L > 0)
                CK(h, cudaMemcpy2DAsync(h->d_ts_win, (size_t)h->ts_cap * 4, h->d_ts_win + (lo - h->ts_lo), (size_t)h->ts_cap * 4,
                                        (size_t)L * 4, (size_t)B, cudaMemcpyDeviceToDevice, st));
            h->ts_lo = lo;
        }
        CK(h, cudaMemcpy2DAsync(h->d_ts_win + (h->ts_R - h->ts_lo), (size_t)h->ts_cap * 4, in + off, (size_t)in_stride * 4,
                                (size_t)s * 4, (size_t)B, cudaMemcpyDeviceToDevice, st));
        h->ts_R += s;
        off += s;
        if ((rc = ts_advance(h, 0, out ? out + (h->ts_ha - ha0) * H : nullptr, out_stride, st))) {
            ts_release(h);
            return rc;
        }
    }
    return B200GATE_OK;
}

int b200gate_tstream_finish(b200gate_handle* h, float* out, int64_t out_stride, int64_t out_capacity, int64_t* n_out,
                            void* stream) {
    if (!h) return B200GATE_ERR_ARG;
    if (!h->ts_open) return fail(h, B200GATE_ERR_STATE, "no open torch stream (b200gate_tstream_begin first)");
    if (!n_out || out_capacity < 0 || (out_capacity > 0 && !out) || (h->ts_B > 1 && out_stride < out_capacity))
        return fail(h, B200GATE_ERR_ARG, "bad argument");
    if (h->ts_mode == 2) return fail(h, B200GATE_ERR_STATE, kTsPerRow);
    const long long H = h->p.hop_length, R = h->ts_R;
    if (R < 2 * h->p.win_length) return fail(h, B200GATE_ERR_ARG, "x must be bigger than %d", 2 * h->p.win_length);
    const long long T = R / H + 1, m = (T + 1 - h->ts_ha) * H;      // the rest of torch.istft's (T - 1) H samples
    if (out_capacity < m)
        return fail(h, B200GATE_ERR_ARG, "out_capacity %lld < %lld samples returned by finish", (long long)out_capacity, m);
    *n_out = m;
    const int rc = ts_advance(h, T, out, out_stride, (cudaStream_t)stream);
    ts_release(h);                                            // (cudaFree waits for the device)
    return rc;
}

int b200gate_tstream_push_rows(b200gate_handle* h, const float* in, const int64_t* n, int64_t in_stride, float* out,
                               int64_t out_stride, int64_t out_capacity, int64_t* n_out, void* stream) {
    if (!h) return B200GATE_ERR_ARG;
    int rc;
    if ((rc = sess_check(h))) return rc;
    const long long B = h->ts_B, H = h->p.hop_length, S = h->ts_slice;
    if (!n || !n_out || out_capacity < 0 || (out_capacity > 0 && !out) || (B > 1 && out_stride < out_capacity))
        return fail(h, B200GATE_ERR_ARG, "bad argument");
    long long n_max = 0, m_max = 0;
    for (long long b = 0; b < B; ++b) {
        if (n[b] < 0) return fail(h, B200GATE_ERR_ARG, "row %lld: a negative sample count (%lld)", b, (long long)n[b]);
        n_max = std::max(n_max, (long long)n[b]);
        m_max = std::max(m_max, (ts_hops_done(h, h->ts_row[b].R + n[b]) - h->ts_row[b].ha) * H);
    }
    if (n_max > 0 && (!in || (B > 1 && in_stride < n_max))) return fail(h, B200GATE_ERR_ARG, "bad argument");
    if (out_capacity < m_max)
        return fail(h, B200GATE_ERR_ARG, "out_capacity %lld < %lld samples returned by this push", (long long)out_capacity, m_max);
    for (long long b = 0; b < B; ++b) n_out[b] = (ts_hops_done(h, h->ts_row[b].R + n[b]) - h->ts_row[b].ha) * H;
    h->ts_mode = 2;
    cudaStream_t st = (cudaStream_t)stream;
    std::vector<long long>& y0 = h->ts_y0;               // row b's output sample j goes to out[y0[b] + j] in this call
    for (long long b = 0; b < B; ++b) y0[b] = b * out_stride - (h->ts_row[b].ha - 2) * H;
    for (long long off = 0; off < n_max; off += S) {
        int k;
        SessRow* tab = sess_slot(h, &k);
        TsSlice span{};
        span.Tb = INT_MAX;
        for (long long b = 0; b < B; ++b) {
            b200gate_handle::TsRow& r = h->ts_row[b];
            const long long s = std::max(0LL, std::min(S, (long long)n[b] - off));
            if (s == 0) continue;
            SessRow& e = tab[b];
            e.n = (int)s;
            e.keep = r.R - r.lo;
            if (r.R - r.lo + s > h->ts_cap) {               // compact: keep the samples of frames nA on
                const long long lo = std::max(0LL, r.nA * H - kN / 2);
                e.keep = r.R - lo;
                e.shift = lo - r.lo;
                r.lo = lo;
            }
            r.R += s;
            sess_fill(h, r, e, 0, y0[b], span);
        }
        if ((rc = sess_submit(h, k, span, in, in_stride, off, out, st))) {
            ts_release(h);
            return rc;
        }
    }
    return B200GATE_OK;
}

int b200gate_tstream_end_rows(b200gate_handle* h, const int64_t* rows, int64_t k, float* out, int64_t out_stride,
                              int64_t out_capacity, int64_t* n_out, void* stream) {
    if (!h) return B200GATE_ERR_ARG;
    int rc;
    if ((rc = sess_check(h))) return rc;
    if ((k > 0 && !n_out) || out_capacity < 0 || (out_capacity > 0 && !out) || (k > 1 && out_stride < out_capacity))
        return fail(h, B200GATE_ERR_ARG, "bad argument");
    if ((rc = sess_check_rows(h, rows, k))) return rc;
    const long long H = h->p.hop_length;
    long long m_max = 0;
    for (int64_t i = 0; i < k; ++i) {
        const b200gate_handle::TsRow& r = h->ts_row[rows[i]];
        if (r.R < 2 * h->p.win_length)
            return fail(h, B200GATE_ERR_ARG, "x must be bigger than %d (row %lld holds %lld samples)", 2 * h->p.win_length,
                        (long long)rows[i], r.R);
        m_max = std::max(m_max, (r.R / H + 2 - r.ha) * H);     // the rest of torch.istft's (R / H) H samples
    }
    if (out_capacity < m_max)
        return fail(h, B200GATE_ERR_ARG, "out_capacity %lld < %lld samples returned by end", (long long)out_capacity, m_max);
    if (k == 0) return B200GATE_OK;
    h->ts_mode = 2;
    int slot;
    SessRow* tab = sess_slot(h, &slot);
    TsSlice span{};
    span.Tb = INT_MAX;
    for (int64_t i = 0; i < k; ++i) {
        b200gate_handle::TsRow& r = h->ts_row[rows[i]];
        n_out[i] = (r.R / H + 2 - r.ha) * H;
        sess_fill(h, r, tab[rows[i]], r.R / H + 1, i * out_stride - (r.ha - 2) * H, span);
        r = b200gate_handle::TsRow{};                         // the row's next samples start a new session
    }
    if ((rc = sess_submit(h, slot, span, nullptr, 0, 0, out, (cudaStream_t)stream))) ts_release(h);
    return rc;
}

int b200gate_tstream_reset_rows(b200gate_handle* h, const int64_t* rows, int64_t k) {
    if (!h) return B200GATE_ERR_ARG;
    int rc;
    if ((rc = sess_check(h)) || (rc = sess_check_rows(h, rows, k))) return rc;
    h->ts_mode = 2;
    for (int64_t i = 0; i < k; ++i) h->ts_row[rows[i]] = b200gate_handle::TsRow{};
    return B200GATE_OK;
}


int b200gate_torch_apply_masks(b200gate_handle* h, const void* in, void* out, int dtype, int64_t C, int64_t N, int64_t in_stride,
                               int64_t out_stride, int is_device, void* stream) {
    if (!h) return B200GATE_ERR_ARG;
    if (h->ts_open) return fail(h, B200GATE_ERR_STATE, kTsOpen);
    if (h->p.surface != B200GATE_SURFACE_TORCH) return fail(h, B200GATE_ERR_STATE, "torch surface only");
    if (!h->masks_valid || h->masks_C != C || h->masks_N != N)
        return fail(h, B200GATE_ERR_STATE, "no masks of a matching forward are kept (run b200gate_run on [%lld][%lld] first; "
                    "tuned n_fft=1024 geometry, one workspace batch)", (long long)C, (long long)N);
    h->reuse_masks = true;
    const int rc = b200gate_run(h, in, out, dtype, C, N, in_stride, out_stride, is_device, stream);
    h->reuse_masks = false;
    return rc;
}

int b200gate_torch_apply_masks_rows(b200gate_handle* h, const b200gate_row* rows, int64_t n_rows, int dtype, int is_device,
                                    void* stream) {
    if (!h) return B200GATE_ERR_ARG;
    if (h->ts_open) return fail(h, B200GATE_ERR_STATE, kTsOpen);
    if (h->p.surface != B200GATE_SURFACE_TORCH) return fail(h, B200GATE_ERR_STATE, "torch surface only");
    if (!rows || n_rows <= 0) return fail(h, B200GATE_ERR_ARG, "bad argument");
    bool match = h->masks_valid && (int64_t)h->masks_rows_n.size() == n_rows;
    for (int64_t r = 0; match && r < n_rows; ++r) match = rows[r].n == h->masks_rows_n[(size_t)r];
    if (!match)
        return fail(h, B200GATE_ERR_STATE, "no masks of a matching forward are kept (run b200gate_run_rows on %lld rows of the "
                    "same lengths first; one workspace batch)", (long long)n_rows);
    h->reuse_masks = true;
    const int rc = b200gate_run_rows(h, rows, n_rows, dtype, is_device, stream);
    h->reuse_masks = false;
    return rc;
}

// ---- multi-GPU: kernel-issued NVLink stores (gate_peer.cuh) ---------------------------------------------------------
int b200gate_peer_push(const void* src, void* const* peer_dst, int32_t n_peers, int64_t rows, int64_t row_bytes,
                       int64_t src_stride_bytes, int64_t dst_stride_bytes, int32_t n_ctas, void* stream) {
    if (!src || !peer_dst || n_peers < 0 || n_peers > kMaxPeers || rows < 0 || row_bytes < 0) return B200GATE_ERR_ARG;
    if (n_peers == 0 || rows == 0 || row_bytes == 0) return B200GATE_OK;
    if ((row_bytes | src_stride_bytes | dst_stride_bytes | (int64_t)(uintptr_t)src) & 15) return B200GATE_ERR_ARG;
    PushArgs a{};
    a.src = (const uint4*)src;
    for (int p = 0; p < n_peers; ++p) {
        if (!peer_dst[p] || ((uintptr_t)peer_dst[p] & 15)) return B200GATE_ERR_ARG;
        a.dst[p] = (uint4*)peer_dst[p];
    }
    a.n_dst = n_peers;
    a.rows = rows; a.vec_per_row = row_bytes / 16; a.src_stride = src_stride_bytes / 16; a.dst_stride = dst_stride_bytes / 16;
    const int ctas = n_ctas > 0 ? n_ctas : 12;
    static bool attr_set = false;
    if (!attr_set) { cudaFuncSetAttribute(k_peer_push, cudaFuncAttributeMaxDynamicSharedMemorySize, kPushSmemBytes); attr_set = true; }
    B200_LAUNCH(k_peer_push, dim3(ctas), dim3(kPushThreads), kPushSmemBytes, (cudaStream_t)stream, a);
    return cudaGetLastError() == cudaSuccess ? B200GATE_OK : B200GATE_ERR_CUDA;
}

int b200gate_peer_barrier(void* local_flags, void* const* peer_flags, int32_t rank, int32_t world, uint32_t epoch, void* stream) {
    if (!local_flags || !peer_flags || world < 1 || world > kMaxPeers || rank < 0 || rank >= world) return B200GATE_ERR_ARG;
    BarrierArgs a{};
    a.local_flags = (unsigned*)local_flags;
    for (int p = 0; p < world; ++p) a.peer_flags[p] = (unsigned*)peer_flags[p];
    a.rank = rank; a.world = world; a.epoch = epoch;
    B200_LAUNCH(k_peer_barrier, dim3(1), dim3(32), 0, (cudaStream_t)stream, a);
    return cudaGetLastError() == cudaSuccess ? B200GATE_OK : B200GATE_ERR_CUDA;
}

int b200gate_run_sharded(b200gate_handle* h, const void* in_local, int dtype, int64_t C_local, int64_t N, int64_t in_stride,
                         void* gathered_local, void* const* gathered_peers, void* flags_local, void* const* flags_peers,
                         uint32_t epoch, int32_t rank, int32_t world, int32_t groups, int32_t push_ctas,
                         void* compute_stream, void* comm_stream) {
    if (!h || !in_local || !gathered_local || world < 1 || world > kMaxPeers || rank < 0 || rank >= world || C_local <= 0)
        return fail(h, B200GATE_ERR_ARG, "bad argument");
    if (world > 1 && (!gathered_peers || !flags_local || !flags_peers || !comm_stream || comm_stream == compute_stream))
        return fail(h, B200GATE_ERR_ARG, "a sharded run needs peer mappings, flag arrays and a separate communication stream");
    const size_t es = dtype_size(dtype);
    if (es == 0) return fail(h, B200GATE_ERR_ARG, "bad dtype");
    cudaStream_t cs = (cudaStream_t)compute_stream, ms = (cudaStream_t)comm_stream;
    if (groups < 1) groups = 1;
    const int64_t gs = (C_local + groups - 1) / groups;
    while (h->group_ev.size() < (size_t)groups + 1) {
        cudaEvent_t e;
        CK(h, cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        h->group_ev.push_back(e);
    }
    // the previous step's pushes (other ranks') may still be landing in OUR buffer only before their barrier; ours are
    // ordered by the communication stream itself.  Compute must not overwrite rows a previous push is still reading:
    CK(h, cudaEventRecord(h->group_ev[groups], ms));
    CK(h, cudaStreamWaitEvent(cs, h->group_ev[groups], 0));
    char* mine = (char*)gathered_local + (size_t)rank * C_local * N * es;
    int gi = 0;
    for (int64_t g0 = 0; g0 < C_local; g0 += gs, ++gi) {
        const int64_t g1 = std::min<int64_t>(C_local, g0 + gs);
        const int rc = b200gate_run(h, (const char*)in_local + (size_t)g0 * in_stride * es, mine + (size_t)g0 * N * es, dtype,
                                    g1 - g0, N, in_stride, N, 1, compute_stream);
        if (rc) return rc;
        if (world == 1) continue;
        CK(h, cudaEventRecord(h->group_ev[gi], cs));
        CK(h, cudaStreamWaitEvent(ms, h->group_ev[gi], 0));
        void* dst[kMaxPeers];
        int np = 0;
        for (int p = 0; p < world; ++p)
            if (p != rank) dst[np++] = (char*)gathered_peers[p] + ((size_t)rank * C_local + g0) * N * es;
        const int rc2 = b200gate_peer_push(mine + (size_t)g0 * N * es, dst, np, g1 - g0, (int64_t)(N * es), (int64_t)(N * es),
                                           (int64_t)(N * es), push_ctas, comm_stream);
        if (rc2) return fail(h, rc2, "peer push failed (rows must be 16-byte multiples)");
    }
    if (world > 1) {
        const int rc = b200gate_peer_barrier(flags_local, flags_peers, rank, world, epoch, comm_stream);
        if (rc) return fail(h, rc, "peer barrier failed");
        CK(h, cudaEventRecord(h->group_ev[groups], ms));
        CK(h, cudaStreamWaitEvent(cs, h->group_ev[groups], 0));
    }
    return B200GATE_OK;
}

}  // extern "C"
