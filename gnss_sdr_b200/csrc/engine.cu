// Host side of libb200gnss.so: engine, IQ band stores, channel registry and the tracking C ABI.
// The shapes mirror the reference's correlator class
// (src/algorithms/tracking/libs/cpu_multicorrelator_real_codes.{h,cc}); see include/b200gnss.h
// for the per-function citations.

#include "common.cuh"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <new>
#include <vector>

namespace b200
{
static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
const char* get_error() { return g_err; }

}  // namespace b200

#include "engine.cuh"

using namespace b200;

namespace b200
{
int upload_tables(b200_engine* e)
{
    if (!e->tables_dirty) return B200_OK;
    BandDesc bd[kMaxBands];
    for (int i = 0; i < kMaxBands; i++)
        {
            bd[i].base = e->bands[i].base;
            bd[i].mask = e->bands[i].mask;
            bd[i].first_index = e->bands[i].first_index;
            bd[i].limit = e->bands[i].capacity;
            bd[i].fmt = e->bands[i].fmt;
        }
    B200_CUDA_TRY(cudaMemcpyAsync(e->bands_dev, bd, sizeof(bd), cudaMemcpyHostToDevice, e->stream));
    const int n = static_cast<int>(e->chans.size());
    B200_CUDA_TRY(e->chans_dev.grow(n, n + 64));
    e->max_code_len = 0;
    e->taps_mask = 0u;
    e->fmt_mask = 0u;
    e->any_high_dyn = false;
    if (n > 0)
        {
            std::vector<ChanDesc> cd(n);
            for (int i = 0; i < n; i++)
                {
                    cd[i] = e->chans[i].desc;
                    if (cd[i].code_len > e->max_code_len) e->max_code_len = cd[i].code_len;
                    if (cd[i].code == nullptr) continue;
                    if (cd[i].high_dyn) e->any_high_dyn = true;
                    e->taps_mask |= 1u << cd[i].taps;
                    e->fmt_mask |= 1u << e->bands[cd[i].band].fmt;
                }
            // synchronous-safe: source is a temporary, so block until the copy has been staged
            B200_CUDA_TRY(cudaMemcpyAsync(e->chans_dev, cd.data(), sizeof(ChanDesc) * n, cudaMemcpyHostToDevice, e->stream));
            B200_CUDA_TRY(cudaStreamSynchronize(e->stream));
        }
    e->tables_dirty = false;
    return B200_OK;
}

int ensure_partials(b200_engine* e, int n_items, int slices)
{
    if (slices <= 1) return B200_OK;
    const size_t need = trk_partial_elems(n_items, slices);
    B200_CUDA_TRY(e->partial.grow(need, need + need / 4));
    if (!e->counters.fits(n_items))
        {
            B200_CUDA_TRY(e->counters.alloc(n_items + n_items / 4 + 16));
            B200_CUDA_TRY(cudaMemsetAsync(e->counters, 0, sizeof(unsigned int) * e->counters.capacity(), e->stream));
        }
    return B200_OK;
}

// few items: split epochs into slices so the whole chip works on them
int batch_slices(int n_items)
{
    int slices = 1;
    if (n_items < 592) slices = (592 + n_items - 1) / n_items;
    if (slices > 64) slices = 64;
    return slices;
}

unsigned long long next_pow2(unsigned long long v)
{
    unsigned long long p = 2;
    while (p < v) p <<= 1;
    return p;
}

// FileSourceBase::itemTypeToSize (file_source_base.cc:340-378): the complex item types, as interleaved (I, Q) pairs
const char* const kItemTypes[] = {nullptr, "ibyte", "ishort", nullptr, "gr_complex"};

const char* item_type_name(SampleFormat f) { return kItemTypes[f]; }

// B200_OK and *f, or B200_ERR_ARG with the error text for a type that is not one of kItemTypes
int parse_item_type(const char* item_type, const char* caller, SampleFormat* f)
{
    for (const SampleFormat k : {kCf32, kI16, kI8})
        if (item_type && std::strcmp(item_type, kItemTypes[k]) == 0)
            {
                *f = k;
                return B200_OK;
            }
    set_error("%s: item type %s is not an interleaved complex type (gr_complex, ishort, ibyte)", caller, item_type ? item_type : "(null)");
    return B200_ERR_ARG;
}

// A float band takes every push (integers are widened on the way in); a narrow band only pushes of its own type, which are
// copied as they are.  Otherwise B200_ERR_STATE with the error text.
int check_push_format(const Band& b, int band, SampleFormat f)
{
    if (b.fmt == kCf32 || f == b.fmt) return B200_OK;
    set_error("band %d holds %s samples: a %s push cannot be written into it", band, item_type_name(b.fmt), item_type_name(f));
    return B200_ERR_STATE;
}
}  // namespace

extern "C"
{
    int b200_version(void) { return 100; }
    const char* b200_last_error(void) { return get_error(); }

    int b200_device_count(int* count)
    {
        if (!count) return B200_ERR_ARG;
        int n = 0;
        cudaError_t err = cudaGetDeviceCount(&n);
        if (err != cudaSuccess)
            {
                set_error("cudaGetDeviceCount: %s", cudaGetErrorString(err));
                *count = 0;
                return B200_ERR_NODEV;
            }
        *count = n;
        return B200_OK;
    }

    int b200_engine_create(b200_engine** out, int device, void* stream)
    {
        if (!out) return B200_ERR_ARG;
        *out = nullptr;
        int n = 0;
        if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0)
            {
                set_error("no CUDA device visible");
                return B200_ERR_NODEV;
            }
        if (device < 0 || device >= n)
            {
                set_error("device %d out of range (have %d)", device, n);
                return B200_ERR_ARG;
            }
        cudaDeviceProp prop{};
        B200_CUDA_TRY(cudaGetDeviceProperties(&prop, device));
        if (prop.major != 9 || prop.minor != 0)
            {
                set_error("device %d is sm_%d%d; this library is built for sm_90a only", device, prop.major, prop.minor);
                return B200_ERR_NODEV;
            }
        B200_ENTER_DEVICE(device);
        std::unique_ptr<b200_engine> e(new (std::nothrow) b200_engine());
        if (!e) return B200_ERR_NOMEM;
        e->device = device;
        if (stream)
            e->stream.borrow(static_cast<cudaStream_t>(stream));
        else
            B200_CUDA_TRY(e->stream.create(cudaStreamNonBlocking));
        B200_CUDA_TRY(e->copy_stream.create(cudaStreamNonBlocking));
        B200_CUDA_TRY(e->copy_done.create(cudaEventDisableTiming));
        B200_CUDA_TRY(e->t0.create(cudaEventDefault));
        B200_CUDA_TRY(e->t1.create(cudaEventDefault));
        B200_CUDA_TRY(e->bands_dev.alloc(kMaxBands));
        *out = e.release();
        return B200_OK;
    }

    int b200_engine_destroy(b200_engine* e)
    {
        if (!e) return B200_ERR_ARG;
        cudaSetDevice(e->device);
        delete e;
        return B200_OK;
    }

    int b200_engine_sync(b200_engine* e)
    {
        if (!e) return B200_ERR_ARG;
        B200_CUDA_TRY(cudaStreamSynchronize(e->copy_stream));
        B200_CUDA_TRY(cudaStreamSynchronize(e->stream));
        return B200_OK;
    }

    int b200_engine_timer_start(b200_engine* e)
    {
        if (!e) return B200_ERR_ARG;
        B200_CUDA_TRY(cudaEventRecord(e->t0, e->stream));
        return B200_OK;
    }

    int b200_engine_timer_stop_ms(b200_engine* e, float* ms)
    {
        if (!e || !ms) return B200_ERR_ARG;
        B200_CUDA_TRY(cudaEventRecord(e->t1, e->stream));
        B200_CUDA_TRY(cudaEventSynchronize(e->t1));
        B200_CUDA_TRY(cudaEventElapsedTime(ms, e->t0, e->t1));
        return B200_OK;
    }

    int b200_engine_launch_count(b200_engine* e, uint64_t* n)
    {
        if (!e || !n) return B200_ERR_ARG;
        *n = e->launches.load();
        return B200_OK;
    }

    // ---- signal conditioners (b200_iq_set_conditioner) ------------------------------------------------------------
    static unsigned long long ceil_div(unsigned long long a, unsigned long long d) { return a / d + (a % d != 0); }

    // the largest tap count among the conditioners that read `band` (0: none feeds from it)
    static unsigned conditioner_taps(const b200_engine* e, int band)
    {
        unsigned t = 0;
        for (const Band& d : e->bands)
            if (d.cond.src == band) t = std::max(t, d.cond.n_taps);
        return t;
    }

    // caller holds e->mu: the window of a conditioned band follows its source's: write_index = ceil(src write_index / D),
    // valid_from = 0 at stream start, else ceil((src valid_from + T - 1) / D), never below cond.floor nor above write_index
    static void conditioned_window(b200_engine* e, Band& d)
    {
        const Band& s = e->bands[d.cond.src];
        const unsigned long long dec = d.cond.decimation;
        d.write_index = ceil_div(s.write_index, dec);
        const unsigned long long rule = s.valid_from == 0 ? 0 : ceil_div(s.valid_from + d.cond.n_taps - 1, dec);
        d.valid_from = std::min(std::max(rule, d.cond.floor), d.write_index);
    }

    // caller holds e->mu: the source `band` moved its valid_from (a push_at gap or restart, b200_iq_forget): its
    // destinations' windows follow, and a restarted stream is valid again from its own start
    static void source_restarted(b200_engine* e, int band)
    {
        for (Band& d : e->bands)
            if (d.cond.src == band)
                {
                    d.cond.floor = 0;
                    conditioned_window(e, d);
                }
    }

    // caller holds e->mu: `band` (re-created or attached) is neither end of a conditioner any more
    static void drop_conditioners(b200_engine* e, int band)
    {
        e->bands[band].cond.src = -1;
        for (Band& d : e->bands)
            if (d.cond.src == band) d.cond.src = -1;
    }

    static int record_cond_done(Band& b, cudaStream_t st)
    {
        if (!b.cond_done) B200_CUDA_TRY(b.cond_done.create(cudaEventDisableTiming));
        B200_CUDA_TRY(cudaEventRecord(b.cond_done, st));
        b.cond_recorded = true;
        return B200_OK;
    }

    // caller holds e->mu: `band` has been written up to its write_index from old_write.  Each conditioner that reads it
    // launches once for its newly complete outputs [ceil(old_write / D), ceil(write_index / D)) on the compute stream, and
    // cond_done marks that launch on its destination and the last one on the source.  No conditioner: nothing is issued.
    static int run_conditioners(b200_engine* e, int band, unsigned long long old_write)
    {
        Band& s = e->bands[band];
        bool launched = false;
        for (Band& d : e->bands)
            {
                if (d.cond.src != band) continue;
                const unsigned long long dec = d.cond.decimation, j0 = ceil_div(old_write, dec), j1 = ceil_div(s.write_index, dec);
                if (j1 > j0)
                    {
                        const int rc = launch_iq_condition(s.dev, s.fmt, s.mask, d.cond.taps, static_cast<int>(d.cond.n_taps), static_cast<int>(dec), j0,
                            j1 - j0, d.cond.real_taps, d.cond.rot_hi, d.cond.rot_lo, reinterpret_cast<float2*>(d.dev.get()), d.mask, e->stream);
                        if (rc) return rc;
                        e->launches++;
                        if (const int rc2 = record_cond_done(d, e->stream)) return rc2;
                        launched = true;
                    }
                conditioned_window(e, d);
            }
        return launched ? record_cond_done(s, e->stream) : B200_OK;
    }

    // B200_OK, or B200_ERR_STATE with the error text when a conditioner fills `band`
    static int check_not_conditioned(const Band& b, int band)
    {
        if (b.cond.src < 0) return B200_OK;
        set_error("band %d is filled by its conditioner from band %d: it takes no pushes of its own", band, b.cond.src);
        return B200_ERR_STATE;
    }

    // ---- bands -----------------------------------------------------------------------------
    // caller holds e->mu; before the band is re-created or attached: queued launches may still read its owned ring
    static int release_owned_ring(b200_engine* e, Band& b)
    {
        if (!b.dev) return B200_OK;
        B200_ENTER_DEVICE(e->device);
        B200_CUDA_TRY(cudaStreamSynchronize(e->stream));
        B200_CUDA_TRY(b.dev.reset());
        return B200_OK;
    }

    int b200_iq_create(b200_engine* e, int band, uint64_t capacity_samples)
    {
        return b200_iq_create_typed(e, band, capacity_samples, "gr_complex");
    }

    int b200_iq_create_typed(b200_engine* e, int band, uint64_t capacity_samples, const char* item_type)
    {
        if (!e || band < 0 || band >= kMaxBands || capacity_samples == 0) return B200_ERR_ARG;
        SampleFormat fmt;
        if (const int rc = parse_item_type(item_type, "iq_create_typed", &fmt)) return rc;
        std::lock_guard<std::mutex> lk(e->mu);
        B200_ENTER_DEVICE(e->device);
        Band& b = e->bands[band];
        if (const int rc = release_owned_ring(e, b)) return rc;
        drop_conditioners(e, band);
        const unsigned long long cap = next_pow2(capacity_samples);
        cudaError_t err = b.dev.alloc(cap * 2ULL * fmt);
        if (err != cudaSuccess)
            {
                set_error("band %d: device allocation of %llu %s samples: %s", band, cap, item_type, cudaGetErrorString(err));
                return B200_ERR_NOMEM;
            }
        b.base = b.dev;
        b.fmt = fmt;
        b.capacity = cap;
        b.mask = cap - 1;
        b.first_index = 0;
        b.write_index = 0;
        b.valid_from = 0;
        b.attached = false;
        b.in_use = true;
        e->tables_dirty = true;
        return B200_OK;
    }

    // n items of item_bytes from host into the slots [off, off + n) of a device ring of cap items (split at its end), on the
    // copy stream; copy_done marks the copy and the compute stream waits for it, so every later launch sees the samples and a
    // band search (acq_engine.cu, band_input) can wait for them alone.  n == 0 queues nothing.
    static int copy_in(b200_engine* e, void* ring, unsigned long long cap, unsigned long long off, const void* host, unsigned long long n,
        size_t item_bytes)
    {
        if (n == 0) return B200_OK;
        char* const dst = static_cast<char*>(ring);
        const char* const src = static_cast<const char*>(host);
        const unsigned long long first = std::min(n, cap - off);
        B200_CUDA_TRY(cudaMemcpyAsync(dst + off * item_bytes, src, first * item_bytes, cudaMemcpyHostToDevice, e->copy_stream));
        if (n > first) B200_CUDA_TRY(cudaMemcpyAsync(dst, src + first * item_bytes, (n - first) * item_bytes, cudaMemcpyHostToDevice, e->copy_stream));
        B200_CUDA_TRY(cudaEventRecord(e->copy_done, e->copy_stream));
        B200_CUDA_TRY(cudaStreamWaitEvent(e->stream, e->copy_done, 0));
        return B200_OK;
    }

    // The one write path of an owned ring: n host samples of format fmt at the band's write index.  Samples of the ring's own
    // format are copied into it; integers pushed into a float ring cross PCIe as they are and are converted into the ring on
    // the device; anything else is refused before a byte is written (check_push_format).  (Overwriting samples
    // that an in-flight launch still reads is the caller's ring-sizing responsibility, exactly as with any circular sample
    // buffer.)
    static int push_samples(b200_engine* e, int band, const void* host, uint64_t n, SampleFormat fmt, uint64_t* first_index)
    {
        if (!e || band < 0 || band >= kMaxBands || (!host && n)) return B200_ERR_ARG;
        std::lock_guard<std::mutex> lk(e->mu);
        Band& b = e->bands[band];
        if (const int rc = b.check_owned_ring(band)) return rc;
        if (const int rc = check_push_format(b, band, fmt)) return rc;
        if (const int rc = check_not_conditioned(b, band)) return rc;
        if (n > b.capacity)
            {
                set_error("push of %llu samples exceeds ring capacity %llu", (unsigned long long)n, b.capacity);
                return B200_ERR_RANGE;
            }
        if (const unsigned taps = conditioner_taps(e, band))
            if (n > b.capacity - (taps - 1))
                {
                    set_error("push of %llu samples into band %d: its conditioners' %u-tap history must stay in the ring, at most %llu per push",
                        (unsigned long long)n, band, taps, b.capacity - (taps - 1));
                    return B200_ERR_RANGE;
                }
        B200_ENTER_DEVICE(e->device);
        if (first_index) *first_index = b.write_index;
        if (n == 0) return B200_OK;
        const unsigned long long old_write = b.write_index;
        if (fmt == b.fmt)
            {
                // slots that a conditioner launch queued by an earlier push still reads are overwritten only after it
                if (b.cond_recorded) B200_CUDA_TRY(cudaStreamWaitEvent(e->copy_stream, b.cond_done, 0));
                const int rc = copy_in(e, b.dev, b.capacity, b.write_index & b.mask, host, n, 2 * static_cast<size_t>(fmt));
                if (rc) return rc;
            }
        else
            {
                // raw integers cross PCIe on the copy stream; the conversion into the float ring runs on the compute
                // stream (ordered before every later correlator launch), so the copy engine goes straight on to the
                // next block, which lands in the other staging buffer
                const unsigned long long bytes = n * 2ULL * static_cast<unsigned long long>(fmt);
                const int k = b.raw_next;
                b.raw_next ^= 1;
                if (!b.raw_free[k]) B200_CUDA_TRY(b.raw_free[k].create(cudaEventDisableTiming));
                if (!b.raw_stage[k].fits(bytes))
                    {
                        B200_CUDA_TRY(cudaStreamSynchronize(e->copy_stream));
                        B200_CUDA_TRY(cudaStreamSynchronize(e->stream));
                        B200_CUDA_TRY(b.raw_stage[k].alloc(bytes + bytes / 4 + 256));
                        B200_CUDA_TRY(cudaEventRecord(b.raw_free[k], e->stream));
                    }
                B200_CUDA_TRY(cudaStreamWaitEvent(e->copy_stream, b.raw_free[k], 0));
                int rc = copy_in(e, b.raw_stage[k], n, 0, host, n, 2 * static_cast<size_t>(fmt));
                if (rc) return rc;
                float2* const ring = reinterpret_cast<float2*>(b.dev.get());
                rc = (fmt == kI16) ? launch_convert_i16(reinterpret_cast<const short*>(b.raw_stage[k].get()), ring, b.mask, b.write_index, n, e->stream)
                                   : launch_convert_i8(reinterpret_cast<const signed char*>(b.raw_stage[k].get()), ring, b.mask, b.write_index, n, e->stream);
                if (rc) return rc;
                e->launches++;
                B200_CUDA_TRY(cudaEventRecord(b.raw_free[k], e->stream));
                b.raw_last = k;
            }
        b.write_index += n;
        return run_conditioners(e, band, old_write);
    }

    int b200_iq_push(b200_engine* e, int band, const b200_cf32* host, uint64_t n, uint64_t* first_index)
    {
        return push_samples(e, band, host, n, kCf32, first_index);
    }

    int b200_iq_push_i16(b200_engine* e, int band, const int16_t* host_iq, uint64_t n, uint64_t* first_index)
    {
        return push_samples(e, band, host_iq, n, kI16, first_index);
    }

    int b200_iq_push_i8(b200_engine* e, int band, const int8_t* host_iq, uint64_t n, uint64_t* first_index)
    {
        return push_samples(e, band, host_iq, n, kI8, first_index);
    }

    int b200_iq_push_at(b200_engine* e, int band, uint64_t abs_index, const b200_cf32* host, uint64_t n, uint64_t* n_new)
    {
        if (!e || band < 0 || band >= kMaxBands || (!host && n)) return B200_ERR_ARG;
        if (n_new) *n_new = 0;
        // competing producers of one band (every tracking block of a flowgraph sees the same stream and offers the same
        // samples) are serialised here; e->mu itself is only held for the bookkeeping and inside push_samples
        std::lock_guard<std::mutex> plk(e->push_mu[band]);
        uint64_t skip = 0;
        {
            std::lock_guard<std::mutex> lk(e->mu);
            Band& b = e->bands[band];
            if (const int rc = b.check_owned_ring(band)) return rc;
            if (const int rc = check_push_format(b, band, kCf32)) return rc;
            if (const int rc = check_not_conditioned(b, band)) return rc;
            // what the ring holds right now
            const unsigned long long lo = b.window_lo();
            if (abs_index >= lo && abs_index + n <= b.write_index) return B200_OK;  // every sample of this block is already in the band
            if (abs_index > b.write_index || abs_index < lo)
                {
                    // a gap (the first block to track starts long after sample 0) or a stream that starts over at an older
                    // index (a new capture, a test): what the ring held is history, the band restarts at abs_index
                    b.valid_from = abs_index;
                    b.write_index = abs_index;
                    source_restarted(e, band);
                }
            skip = b.write_index - abs_index;
        }
        const int rc = push_samples(e, band, host + skip, n - skip, kCf32, nullptr);
        if (rc == B200_OK && n_new) *n_new = n - skip;
        return rc;
    }

    int b200_iq_forget(b200_engine* e, int band)
    {
        if (!e || band < 0 || band >= kMaxBands) return B200_ERR_ARG;
        std::lock_guard<std::mutex> plk(e->push_mu[band]);
        std::lock_guard<std::mutex> lk(e->mu);
        Band& b = e->bands[band];
        if (!b.in_use || b.attached) return B200_ERR_STATE;
        b.valid_from = b.write_index;
        if (b.cond.src >= 0) b.cond.floor = b.write_index;
        source_restarted(e, band);
        return B200_OK;
    }

    int b200_iq_window(b200_engine* e, int band, uint64_t* valid_from, uint64_t* write_index)
    {
        if (!e || band < 0 || band >= kMaxBands) return B200_ERR_ARG;
        std::lock_guard<std::mutex> lk(e->mu);
        const Band& b = e->bands[band];
        if (!b.in_use) return B200_ERR_STATE;
        if (valid_from) *valid_from = b.window_lo();
        if (write_index) *write_index = b.write_index;
        return B200_OK;
    }

    int b200_iq_push_file(b200_engine* e, int band, const char* path, const char* item_type, uint64_t header_bytes, uint64_t skip_samples,
        uint64_t max_samples, uint64_t chunk_samples, uint64_t* first_index, uint64_t* samples_pushed)
    {
        if (!e || !path || !item_type || band < 0 || band >= kMaxBands) return B200_ERR_ARG;
        SampleFormat fmt;
        if (const int rc = parse_item_type(item_type, "iq_push_file", &fmt)) return rc;
        unsigned long long capacity;
        unsigned history;
        {
            std::lock_guard<std::mutex> lk(e->mu);
            const Band& b = e->bands[band];
            if (const int rc = b.check_owned_ring(band)) return rc;
            if (const int rc = check_push_format(b, band, fmt)) return rc;
            capacity = b.capacity;
            history = conditioner_taps(e, band);
        }
        if (chunk_samples == 0) chunk_samples = 1ULL << 20;
        if (chunk_samples > capacity / 2) chunk_samples = capacity / 2 ? capacity / 2 : 1;
        if (history > 1 && chunk_samples > capacity - (history - 1)) chunk_samples = capacity - (history - 1);
        B200_ENTER_DEVICE(e->device);
        FILE* f = std::fopen(path, "rb");
        if (!f)
            {
                set_error("iq_push_file: cannot open %s", path);
                return B200_ERR_STATE;
            }
        const size_t sample_bytes = 2u * static_cast<size_t>(fmt);
        // samplesToSkip (:385-414): header, then whole samples
        if (std::fseek(f, static_cast<long>(header_bytes + skip_samples * sample_bytes), SEEK_SET) != 0)
            {
                std::fclose(f);
                set_error("iq_push_file: cannot seek in %s", path);
                return B200_ERR_RANGE;
            }
        // two pinned staging buffers: the disk read of block k+1 overlaps the host->device copy of block k
        PinBuf<unsigned char> stage[2];
        CudaEvent freed[2];
        int rc = B200_OK;
        for (int k = 0; k < 2 && rc == B200_OK; k++)
            {
                if (stage[k].alloc(chunk_samples * sample_bytes) != cudaSuccess || freed[k].create(cudaEventDisableTiming) != cudaSuccess)
                    {
                        set_error("iq_push_file: pinned staging allocation failed");
                        rc = B200_ERR_NOMEM;
                    }
            }
        uint64_t total = 0;
        bool have_first = false;
        for (int k = 0; rc == B200_OK && (max_samples == 0 || total < max_samples); k ^= 1)
            {
                if (cudaEventSynchronize(freed[k]) != cudaSuccess)  // the copy that last read this buffer has finished
                    {
                        rc = B200_ERR_CUDA;
                        break;
                    }
                uint64_t want = chunk_samples;
                if (max_samples != 0 && max_samples - total < want) want = max_samples - total;
                const size_t got = std::fread(stage[k], sample_bytes, static_cast<size_t>(want), f);
                if (got == 0) break;
                uint64_t first = 0;
                rc = push_samples(e, band, stage[k], got, fmt, &first);
                if (rc != B200_OK) break;
                if (cudaEventRecord(freed[k], e->copy_stream) != cudaSuccess) rc = B200_ERR_CUDA;
                if (!have_first)
                    {
                        have_first = true;
                        if (first_index) *first_index = first;
                    }
                total += got;
                if (got < want) break;  // end of file
            }
        std::fclose(f);
        cudaStreamSynchronize(e->copy_stream);  // before the staging buffers are released
        if (samples_pushed) *samples_pushed = total;
        return rc;
    }

    int b200_iq_attach_dev(b200_engine* e, int band, const b200_cf32* dev, uint64_t n_samples, uint64_t first_index)
    {
        if (!e || band < 0 || band >= kMaxBands || !dev) return B200_ERR_ARG;
        if (reinterpret_cast<uintptr_t>(dev) & 15)
            {
                set_error("attached band must be 16-byte aligned");
                return B200_ERR_ARG;
            }
        std::lock_guard<std::mutex> lk(e->mu);
        Band& b = e->bands[band];
        if (const int rc = release_owned_ring(e, b)) return rc;
        drop_conditioners(e, band);
        b.base = dev;
        b.fmt = kCf32;
        b.capacity = n_samples;
        b.mask = ~0ULL;
        b.first_index = first_index;
        b.write_index = first_index + n_samples;
        b.valid_from = first_index;
        b.attached = true;
        b.in_use = true;
        e->tables_dirty = true;
        return B200_OK;
    }

    int b200_iq_refill(b200_engine* e, int band, const b200_cf32* host, uint64_t n, uint64_t first_index)
    {
        if (!e || band < 0 || band >= kMaxBands || (!host && n)) return B200_ERR_ARG;
        std::lock_guard<std::mutex> lk(e->mu);
        Band& b = e->bands[band];
        if (b.in_use)
            if (const int rc = check_push_format(b, band, kCf32)) return rc;
        if (!b.in_use || !b.attached)
            {
                set_error("band %d is not an attached device buffer (call b200_iq_attach_dev)", band);
                return B200_ERR_STATE;
            }
        if (n > b.capacity)
            {
                set_error("refill of %llu samples exceeds the attached buffer (%llu)", (unsigned long long)n, b.capacity);
                return B200_ERR_RANGE;
            }
        B200_ENTER_DEVICE(e->device);
        // overwriting samples an in-flight launch still reads is the caller's double-buffering responsibility
        const int rc = copy_in(e, const_cast<void*>(b.base), b.capacity, 0, host, n, sizeof(float2));
        if (rc) return rc;
        if (b.first_index != first_index)
            {
                b.first_index = first_index;
                e->tables_dirty = true;
            }
        b.valid_from = first_index;
        b.write_index = first_index + n;
        return B200_OK;
    }

    int b200_iq_read(b200_engine* e, int band, uint64_t abs_index, uint64_t n, void* host)
    {
        if (!e || band < 0 || band >= kMaxBands || (!host && n)) return B200_ERR_ARG;
        std::lock_guard<std::mutex> lk(e->mu);
        const Band& b = e->bands[band];
        if (!b.in_use)
            {
                set_error("band %d holds no samples (call b200_iq_create or b200_iq_attach_dev)", band);
                return B200_ERR_STATE;
            }
        if (!b.holds(abs_index, n))
            {
                set_error("band %d: samples [%llu, %llu) are outside the band's window [%llu, %llu)", band, (unsigned long long)abs_index,
                    (unsigned long long)(abs_index + n), b.window_lo(), b.write_index);
                return B200_ERR_RANGE;
            }
        if (n == 0) return B200_OK;
        B200_ENTER_DEVICE(e->device);
        // every write into a band is ordered before later work on the compute stream (copy_in, conversions, conditioners)
        const size_t item = 2 * static_cast<size_t>(b.fmt);
        const unsigned long long off = (abs_index - b.first_index) & b.mask;
        const unsigned long long first = std::min<unsigned long long>(n, b.capacity - off);
        B200_CUDA_TRY(cudaMemcpyAsync(host, static_cast<const char*>(b.base) + off * item, first * item, cudaMemcpyDeviceToHost, e->stream));
        if (n > first)
            B200_CUDA_TRY(cudaMemcpyAsync(static_cast<char*>(host) + first * item, b.base, (n - first) * item, cudaMemcpyDeviceToHost, e->stream));
        B200_CUDA_TRY(cudaStreamSynchronize(e->stream));
        return B200_OK;
    }

    int b200_iq_set_conditioner(b200_engine* e, int dst_band, int src_band, uint32_t decimation, const float* taps, uint32_t n_taps,
        double intermediate_freq_hz, double sampling_freq_hz)
    {
        if (!e || dst_band < 0 || dst_band >= kMaxBands) return B200_ERR_ARG;
        if (n_taps == 0)
            {
                std::lock_guard<std::mutex> lk(e->mu);
                e->bands[dst_band].cond.src = -1;
                return B200_OK;
            }
        if (src_band < 0 || src_band >= kMaxBands || !taps || decimation < 1 || !(sampling_freq_hz > 0.0) || !std::isfinite(sampling_freq_hz) ||
            !std::isfinite(intermediate_freq_hz))
            {
                set_error("iq_set_conditioner: band %d, decimation %u, taps %s, fs %g Hz, IF %g Hz: bad argument", src_band, decimation,
                    taps ? "set" : "NULL", sampling_freq_hz, intermediate_freq_hz);
                return B200_ERR_ARG;
            }
        if (dst_band == src_band)
            {
                set_error("iq_set_conditioner: band %d cannot condition into itself", dst_band);
                return B200_ERR_ARG;
            }
        if (n_taps > B200_IQ_MAX_CONDITIONER_TAPS || decimation > B200_IQ_MAX_CONDITIONER_DECIMATION)
            {
                set_error("iq_set_conditioner: %u taps, decimation %u: at most %d taps and decimation %d", n_taps, decimation,
                    B200_IQ_MAX_CONDITIONER_TAPS, B200_IQ_MAX_CONDITIONER_DECIMATION);
                return B200_ERR_RANGE;
            }
        std::lock_guard<std::mutex> lk(e->mu);
        Band& d = e->bands[dst_band];
        const Band& s = e->bands[src_band];
        if (const int rc = s.check_owned_ring(src_band)) return rc;
        if (const int rc = d.check_owned_ring(dst_band)) return rc;
        if (d.fmt != kCf32)
            {
                set_error("iq_set_conditioner: band %d holds %s samples: a conditioner writes gr_complex", dst_band, item_type_name(d.fmt));
                return B200_ERR_STATE;
            }
        if (conditioner_taps(e, dst_band) > 0 || s.cond.src >= 0)
            {
                set_error("iq_set_conditioner: band %d -> band %d would chain conditioners", src_band, dst_band);
                return B200_ERR_STATE;
            }
        if (d.capacity * decimation < s.capacity || s.capacity < n_taps)
            {
                set_error("iq_set_conditioner: band %d (%llu samples) must hold band %d's %llu samples decimated by %u, and band %d at least %u taps",
                    dst_band, d.capacity, src_band, s.capacity, decimation, src_band, n_taps);
                return B200_ERR_RANGE;
            }
        B200_ENTER_DEVICE(e->device);
        // c[k] = h[k] e^{+i k w}, w = 2 pi IF / fs, in double, each component rounded once to float
        const double pi = 3.14159265358979323846;
        const double w = 2.0 * pi * intermediate_freq_hz / sampling_freq_hz;
        std::vector<float2> c(n_taps);
        for (uint32_t k = 0; k < n_taps; k++)
            c[k] = make_float2(static_cast<float>(taps[k] * std::cos(k * w)), static_cast<float>(taps[k] * std::sin(k * w)));
        B200_CUDA_TRY(cudaStreamSynchronize(e->stream));  // launches already queued may still read the old taps
        if (!d.cond.taps.fits(n_taps)) B200_CUDA_TRY(d.cond.taps.alloc(n_taps));
        B200_CUDA_TRY(cudaMemcpyAsync(d.cond.taps, c.data(), sizeof(float2) * n_taps, cudaMemcpyHostToDevice, e->stream));
        B200_CUDA_TRY(cudaStreamSynchronize(e->stream));
        d.cond.src = src_band;
        d.cond.decimation = decimation;
        d.cond.n_taps = n_taps;
        d.cond.real_taps = intermediate_freq_hz == 0.0;
        cond_rotator_step(intermediate_freq_hz, sampling_freq_hz, decimation, &d.cond.rot_hi, &d.cond.rot_lo);
        d.cond.floor = ceil_div(s.write_index, decimation);  // set mid-stream: the destination starts empty there
        conditioned_window(e, d);
        return B200_OK;
    }

    // ---- channels ------------------------------------------------------------------------------
    int b200_trk_channel_create(b200_engine* e, int band, int n_correlators, int* channel_id)
    {
        if (!e || !channel_id || band < 0 || band >= kMaxBands) return B200_ERR_ARG;
        if (n_correlators < 1 || n_correlators > B200_MAX_TAPS)
            {
                set_error("n_correlators %d outside 1..%d", n_correlators, B200_MAX_TAPS);
                return B200_ERR_RANGE;
            }
        std::lock_guard<std::mutex> lk(e->mu);
        Channel c;
        c.desc.band = band;
        c.desc.taps = n_correlators;
        c.desc.code = nullptr;
        c.desc.code_len = 0;
        c.desc.high_dyn = 0;
        for (float& s : c.desc.shifts) s = 0.f;
        e->chans.push_back(std::move(c));
        *channel_id = static_cast<int>(e->chans.size()) - 1;
        e->tables_dirty = true;
        return B200_OK;
    }

    int b200_trk_channel_set_code(b200_engine* e, int channel_id, int code_length_chips, const float* local_code_in, const float* shifts_chips, int high_dynamics)
    {
        if (!e || !local_code_in || !shifts_chips || code_length_chips < 1) return B200_ERR_ARG;
        std::lock_guard<std::mutex> lk(e->mu);
        if (channel_id < 0 || channel_id >= static_cast<int>(e->chans.size())) return B200_ERR_ARG;
        B200_ENTER_DEVICE(e->device);
        Channel& c = e->chans[channel_id];
        // a new table may be read by launches already queued: allocate fresh if it must grow
        if (!c.code_dev.fits(code_length_chips))
            {
                B200_CUDA_TRY(cudaStreamSynchronize(e->stream));
                // the old table is released here: until the new one is in place the channel has none
                c.desc.code = nullptr;
                e->tables_dirty = true;
                B200_CUDA_TRY(c.code_dev.alloc(code_length_chips));
            }
        B200_CUDA_TRY(cudaMemcpyAsync(c.code_dev, local_code_in, sizeof(float) * code_length_chips, cudaMemcpyHostToDevice, e->stream));
        B200_CUDA_TRY(cudaStreamSynchronize(e->stream));  // caller's buffer may go away
        c.desc.code = c.code_dev;
        c.desc.code_len = code_length_chips;
        c.desc.high_dyn = high_dynamics ? 1 : 0;
        for (int t = 0; t < c.desc.taps; t++) c.desc.shifts[t] = shifts_chips[t];
        e->tables_dirty = true;
        return B200_OK;
    }

    int b200_trk_channel_set_taps(b200_engine* e, int channel_id, const float* shifts_chips)
    {
        if (!e || !shifts_chips) return B200_ERR_ARG;
        std::lock_guard<std::mutex> lk(e->mu);
        if (channel_id < 0 || channel_id >= static_cast<int>(e->chans.size())) return B200_ERR_ARG;
        Channel& c = e->chans[channel_id];
        bool changed = false;
        for (int t = 0; t < c.desc.taps; t++)
            {
                if (c.desc.shifts[t] != shifts_chips[t]) changed = true;
                c.desc.shifts[t] = shifts_chips[t];
            }
        // the descriptor table is re-uploaded in stream order before the next launch (earlier launches keep the old taps)
        if (changed) e->tables_dirty = true;
        return B200_OK;
    }

    // caller holds e->mu
    // layout_hint: 1 = consecutive items overlap in the band (a receiver's channels on one stream), 0 = they do not (every
    // item reads its own samples: nothing to share, the per-item kernel streams them faster), -1 = unknown (device items)
    static int batch_dev_impl(b200_engine* e, const b200_trk_item* items_dev, int n_items, b200_cf32* out_dev, int out_stride, int slices,
        int layout_hint = -1)
    {
        B200_ENTER_DEVICE(e->device);
        int rc = upload_tables(e);
        if (rc) return rc;
        if (slices < 1) slices = 1;
        rc = ensure_partials(e, n_items, slices);
        if (rc) return rc;
        // the shared-window kernel takes batches whose channels all have 1, 3 or 5 taps and sit on float bands (it reads float2
        // samples: a narrow ring would be read past its end)
        const unsigned int mask = e->taps_mask;
        const bool shared_legal = (mask == (1u << 1) || mask == (1u << 3) || mask == (1u << 5)) && !e->any_high_dyn && slices == 1 &&
                                  e->fmt_mask == (1u << kCf32);
        const bool use_shared = shared_legal && (e->shared_mode == 1 || (e->shared_mode == 2 && n_items >= 1024 && layout_hint != 0 &&
                                                                            e->max_code_len <= trk_shared_max_code_len()));
        uint64_t launched = 0;
        if (use_shared)
            rc = launch_trk_shared(items_dev, n_items, e->chans_dev, e->bands_dev, reinterpret_cast<float2*>(out_dev), out_stride,
                __builtin_ctz(mask), e->stream, launched);
        else
            rc = launch_trk_batch(items_dev, n_items, e->chans_dev, e->bands_dev, reinterpret_cast<float2*>(out_dev), out_stride,
                slices, e->partial, e->counters, e->max_code_len, mask, e->fmt_mask, e->stream, launched);
        if (rc) return rc;
        e->launches += launched;
        return B200_OK;
    }

    int b200_trk_kernel_choice(b200_engine* e, int mode)
    {
        if (!e || mode < -1 || mode > 2) return B200_ERR_ARG;
        std::lock_guard<std::mutex> lk(e->mu);
        e->shared_mode = mode < 0 ? 2 : mode;
        return B200_OK;
    }

    int b200_trk_batch_dev(b200_engine* e, const b200_trk_item* items_dev, int n_items, b200_cf32* out_dev, int out_stride, int slices)
    {
        if (!e || n_items < 0 || (n_items && (!items_dev || !out_dev)) || out_stride < 1) return B200_ERR_ARG;
        if (n_items == 0) return B200_OK;
        std::lock_guard<std::mutex> lk(e->mu);
        return batch_dev_impl(e, items_dev, n_items, out_dev, out_stride, slices);
    }

    int b200_trk_submit(b200_engine* e, const b200_trk_item* items_host, int n_items, int out_stride, uint64_t* ticket)
    {
        if (!e || !ticket || n_items < 1 || !items_host || out_stride < 1) return B200_ERR_ARG;
        // one lock for the whole submission: concurrent submitters (the reference runs one thread per tracking block)
        // queue whole batches, never interleave the item copy of one with the launch of another
        std::lock_guard<std::mutex> lk(e->mu);
        B200_ENTER_DEVICE(e->device);
        for (int i = 0; i < n_items; i++)
            {
                const int ch = items_host[i].channel;
                if (ch < 0 || ch >= static_cast<int>(e->chans.size()) || e->chans[ch].desc.code == nullptr)
                    {
                        set_error("item %d: channel %d has no code table", i, ch);
                        return B200_ERR_STATE;
                    }
                if (e->chans[ch].desc.taps > out_stride)
                    {
                        set_error("item %d: out_stride %d < taps %d", i, out_stride, e->chans[ch].desc.taps);
                        return B200_ERR_ARG;
                    }
                // ring bands: the epoch must lie inside what has been pushed and not yet overwritten
                const Band& b = e->bands[e->chans[ch].desc.band];
                if (b.in_use && !b.attached && items_host[i].n > 0)
                    {
                        const unsigned long long s0 = items_host[i].sample_index, n = static_cast<unsigned long long>(items_host[i].n);
                        if (!b.holds(s0, n))
                            {
                                set_error("item %d: samples [%llu, %llu) are outside the band's window [%llu, %llu)", i, s0, s0 + n, b.window_lo(),
                                    b.write_index);
                                return B200_ERR_RANGE;
                            }
                    }
            }
        b200_engine::Slot* sl = nullptr;
        for (auto& s : e->slots)
            if (!s.busy)
                {
                    sl = &s;
                    break;
                }
        if (!sl)
            {
                set_error("more than %d batches in flight: call b200_trk_wait", b200_engine::kSlots);
                return B200_ERR_STATE;
            }
        // the slot is released again on every early return below (a transient CUDA error must not leak it)
        struct BusyGuard
        {
            b200_engine::Slot* s;
            bool keep{false};
            ~BusyGuard()
            {
                if (!keep) s->busy = false;
            }
        } guard{sl};
        sl->busy = true;
        if (!sl->done) B200_CUDA_TRY(sl->done.create(cudaEventDisableTiming));
        if (!sl->items_ready) B200_CUDA_TRY(sl->items_ready.create(cudaEventDisableTiming));
        B200_CUDA_TRY(sl->items_dev.grow(n_items, n_items + n_items / 2 + 64));
        B200_CUDA_TRY(sl->items_pin.grow(n_items, n_items + n_items / 2 + 64));
        const int out_elems = n_items * out_stride;
        B200_CUDA_TRY(sl->out_dev.grow(out_elems, out_elems + out_elems / 2 + 64));
        B200_CUDA_TRY(sl->out_pin.grow(out_elems, out_elems + out_elems / 2 + 64));
        sl->n_items = n_items;
        sl->out_stride = out_stride;
        // The shared-window kernel serves items 8g..8g+7 from one copy of the samples, so items
        // should be ordered by start sample.  Already-ordered input (the usual epoch-major layout)
        // is copied as is; otherwise sort a permutation and undo it in b200_trk_wait.
        bool sorted = true;
        for (int i = 1; i < n_items && sorted; i++) sorted = items_host[i - 1].sample_index <= items_host[i].sample_index;
        sl->perm.clear();
        if (sorted)
            {
                std::memcpy(sl->items_pin, items_host, sizeof(b200_trk_item) * n_items);
            }
        else
            {
                sl->perm.resize(n_items);
                for (int i = 0; i < n_items; i++) sl->perm[i] = i;
                std::stable_sort(sl->perm.begin(), sl->perm.end(),
                    [&](int a, int b) { return items_host[a].sample_index < items_host[b].sample_index; });
                for (int i = 0; i < n_items; i++) sl->items_pin[i] = items_host[sl->perm[i]];
            }
        const int slices = batch_slices(n_items);
        // Latency path (a handful of channels waiting for their taps, e.g. the block threads behind the coalescer): the
        // kernel reads the work items straight from the pinned host buffer and writes the taps straight into pinned host
        // memory (unified addressing: cudaMallocHost memory is device-accessible at the same address), so the submission
        // is one launch + one event instead of two copies through the copy engine, two events and a stream hop.
        sl->zero_copy = n_items <= 1024;
        if (sl->zero_copy)
            {
                const int rc = batch_dev_impl(e, sl->items_pin, n_items, reinterpret_cast<b200_cf32*>(sl->out_pin.get()), out_stride, slices);
                if (rc) return rc;
                B200_CUDA_TRY(cudaEventRecord(sl->done, e->stream));
            }
        else
            {
                // The work items travel on the COPY stream, queued behind the sample pushes made so far, and the compute
                // stream waits on an event.  Issued on the compute stream instead, this small host->device copy sits in
                // the copy engine's queue until the previous batch's kernel has finished and holds up every sample
                // push queued behind it, which lowers the sustained host->device rate.
                B200_CUDA_TRY(cudaMemcpyAsync(sl->items_dev, sl->items_pin, sizeof(b200_trk_item) * n_items, cudaMemcpyHostToDevice, e->copy_stream));
                B200_CUDA_TRY(cudaEventRecord(sl->items_ready, e->copy_stream));
                B200_CUDA_TRY(cudaStreamWaitEvent(e->stream, sl->items_ready, 0));
                // do the groups of consecutive (sorted) items the shared-window kernel would form really overlap?
                unsigned long long sum_n = 0, sum_hull = 0;
                for (int g = 0; g < n_items; g += 8)
                    {
                        unsigned long long lo = ~0ULL, hi = 0;
                        for (int i = g; i < n_items && i < g + 8; i++)
                            {
                                const b200_trk_item& it = sl->items_pin[i];
                                const unsigned long long a = it.sample_index + (static_cast<unsigned long long>(e->chans[it.channel].desc.band) << 48);
                                lo = a < lo ? a : lo;
                                hi = a + it.n > hi ? a + it.n : hi;
                                sum_n += it.n > 0 ? it.n : 0;
                            }
                        sum_hull += hi - lo;
                    }
                const int layout_hint = (sum_n > 2 * sum_hull) ? 1 : 0;
                const int rc = batch_dev_impl(e, sl->items_dev, n_items, reinterpret_cast<b200_cf32*>(sl->out_dev.get()), out_stride, slices, layout_hint);
                if (rc) return rc;
                B200_CUDA_TRY(cudaMemcpyAsync(sl->out_pin, sl->out_dev, sizeof(float2) * n_items * out_stride, cudaMemcpyDeviceToHost, e->stream));
                B200_CUDA_TRY(cudaEventRecord(sl->done, e->stream));
            }
        sl->ticket = e->next_ticket++;
        *ticket = sl->ticket;
        guard.keep = true;
        return B200_OK;
    }

    int b200_trk_wait(b200_engine* e, uint64_t ticket, b200_cf32* out_host)
    {
        if (!e || !out_host) return B200_ERR_ARG;
        b200_engine::Slot* sl = nullptr;
        {
            std::lock_guard<std::mutex> lk(e->mu);
            for (auto& s : e->slots)
                if (s.busy && s.ticket == ticket) sl = &s;
        }
        if (!sl)
            {
                set_error("unknown ticket %llu", static_cast<unsigned long long>(ticket));
                return B200_ERR_ARG;
            }
        B200_ENTER_DEVICE(e->device);
        B200_CUDA_TRY(cudaEventSynchronize(sl->done));
        if (sl->perm.empty())
            {
                std::memcpy(out_host, sl->out_pin, sizeof(float2) * sl->n_items * sl->out_stride);
            }
        else
            {
                for (int k = 0; k < sl->n_items; k++)
                    std::memcpy(out_host + static_cast<size_t>(sl->perm[k]) * sl->out_stride, sl->out_pin + static_cast<size_t>(k) * sl->out_stride,
                        sizeof(float2) * sl->out_stride);
            }
        std::lock_guard<std::mutex> lk(e->mu);
        sl->busy = false;
        return B200_OK;
    }

    int b200_trk_batch(b200_engine* e, const b200_trk_item* items_host, int n_items, b200_cf32* out_host, int out_stride)
    {
        if (!e || n_items < 0 || (n_items && (!items_host || !out_host)) || out_stride < 1) return B200_ERR_ARG;
        if (n_items == 0) return B200_OK;
        uint64_t ticket = 0;
        int rc = b200_trk_submit(e, items_host, n_items, out_stride, &ticket);
        if (rc) return rc;
        return b200_trk_wait(e, ticket, out_host);
    }
}

// ---- single correlator object (Cpu_Multicorrelator_Real_Codes shape) ----------------------------
struct b200_trk
{
    CudaStream stream;  // declared first, so released after the buffers used on it
    b200_engine* e{nullptr};
    int max_len{0};
    int taps{0};
    int high_dyn{0};
    DevBuf<float2> sig_dev;
    DevBuf<float> code_dev;
    // host-mapped control block: the kernel reads the item and descriptors and writes the taps
    // straight into pinned host memory (no D2H memcpy on the latency path)
    struct Ctl
    {
        b200_trk_item item;
        ChanDesc chan;
        BandDesc band;
        float2 out[B200_MAX_TAPS];
    };
    PinBuf<Ctl> ctl;
    DevBuf<float2> partial;
    DevBuf<unsigned int> counter;
    int slices_cap{0};
    bool have_code{false};
    // legacy variants (trk_variants.cu): complex local code / 16-bit samples and code
    DevBuf<float2> cplx_code_dev;
    int cplx_code_len{0};
    DevBuf<short> code16_dev;
    int code16_len{0};
    DevBuf<short> sig16_dev;
    DevBuf<short> out16_dev;
    DevBuf<float2> out_cplx_dev;
    float var_shifts[B200_MAX_TAPS] = {0};

    ~b200_trk()
    {
        if (stream) cudaStreamSynchronize(stream);
    }
};

namespace
{
// a local code table of n elements into buf: the launches that read the old table finish first, buf is reallocated when it
// must grow, and the copy has landed on return (the caller's buffer may go away)
template <typename T>
int load_code(b200_trk* t, DevBuf<T>& buf, const void* host, size_t n)
{
    B200_CUDA_TRY(cudaStreamSynchronize(t->stream));
    if (!buf.fits(n)) B200_CUDA_TRY(buf.alloc(n));
    B200_CUDA_TRY(cudaMemcpyAsync(buf, host, sizeof(T) * n, cudaMemcpyHostToDevice, t->stream));
    B200_CUDA_TRY(cudaStreamSynchronize(t->stream));
    return B200_OK;
}

// the signal of one correlate call: n samples of sample_bytes from host into dev, queued on t->stream
int stage_signal(b200_trk* t, void* dev, const void* host, int n, size_t sample_bytes)
{
    if (n < 0 || n > t->max_len)
        {
            set_error("signal_length_samples %d outside 0..%d", n, t->max_len);
            return B200_ERR_RANGE;
        }
    B200_ENTER_DEVICE(t->e->device);
    if (n > 0) B200_CUDA_TRY(cudaMemcpyAsync(dev, host, sample_bytes * n, cudaMemcpyHostToDevice, t->stream));
    return B200_OK;
}
}  // namespace

extern "C"
{
    int b200_trk_create(b200_engine* e, b200_trk** out, int max_signal_length_samples, int n_correlators)
    {
        if (!e || !out || max_signal_length_samples < 1) return B200_ERR_ARG;
        if (n_correlators < 1 || n_correlators > B200_MAX_TAPS)
            {
                set_error("n_correlators %d outside 1..%d", n_correlators, B200_MAX_TAPS);
                return B200_ERR_RANGE;
            }
        B200_ENTER_DEVICE(e->device);
        std::unique_ptr<b200_trk> t(new (std::nothrow) b200_trk());
        if (!t) return B200_ERR_NOMEM;
        t->e = e;
        t->max_len = max_signal_length_samples;
        t->taps = n_correlators;
        B200_CUDA_TRY(t->stream.create(cudaStreamNonBlocking));
        B200_CUDA_TRY(t->sig_dev.alloc(static_cast<size_t>(t->max_len) + 2));
        B200_CUDA_TRY(t->ctl.alloc(1, cudaHostAllocMapped));
        std::memset(t->ctl, 0, sizeof(b200_trk::Ctl));
        t->slices_cap = 64;
        B200_CUDA_TRY(t->partial.alloc(trk_partial_elems(1, t->slices_cap)));
        B200_CUDA_TRY(t->counter.alloc(1));
        B200_CUDA_TRY(cudaMemsetAsync(t->counter, 0, sizeof(unsigned int), t->stream));
        *out = t.release();
        return B200_OK;
    }

    int b200_trk_set_high_dynamics_resampler(b200_trk* t, int use_high_dynamics_resampler)
    {
        if (!t) return B200_ERR_ARG;
        t->high_dyn = use_high_dynamics_resampler ? 1 : 0;
        return B200_OK;
    }

    int b200_trk_set_local_code_and_taps(b200_trk* t, int code_length_chips, const float* local_code_in, const float* shifts_chips)
    {
        if (!t || !local_code_in || !shifts_chips || code_length_chips < 1) return B200_ERR_ARG;
        B200_ENTER_DEVICE(t->e->device);
        if (!t->code_dev.fits(code_length_chips)) t->have_code = false;  // load_code releases the old table
        if (const int rc = load_code(t, t->code_dev, local_code_in, code_length_chips)) return rc;
        ChanDesc& c = t->ctl->chan;
        c.code = t->code_dev;
        c.code_len = code_length_chips;
        c.taps = t->taps;
        c.band = 0;
        for (int k = 0; k < t->taps; k++) c.shifts[k] = shifts_chips[k];
        t->have_code = true;
        return B200_OK;
    }

    int b200_trk_set_taps(b200_trk* t, const float* shifts_chips)
    {
        if (!t || !shifts_chips) return B200_ERR_ARG;
        // the descriptor lives in the host-mapped control block the kernel reads at launch; calls on one handle are
        // serialised by the caller and b200_trk_correlate is synchronous, so no launch is in flight here
        for (int k = 0; k < t->taps; k++) t->ctl->chan.shifts[k] = shifts_chips[k];
        return B200_OK;
    }

    int b200_trk_correlate(b200_trk* t, const b200_cf32* sig_in_host,
        float rem_carrier_phase_in_rad, float phase_step_rad, float phase_rate_step_rad,
        float rem_code_phase_chips, float code_phase_step_chips, float code_phase_rate_step_chips,
        int signal_length_samples, b200_cf32* corr_out_host)
    {
        if (!t || !sig_in_host || !corr_out_host) return B200_ERR_ARG;
        if (!t->have_code)
            {
                set_error("correlate before set_local_code_and_taps");
                return B200_ERR_STATE;
            }
        const int n = signal_length_samples;
        if (const int rc = stage_signal(t, t->sig_dev, sig_in_host, n, sizeof(float2))) return rc;
        b200_trk::Ctl* c = t->ctl;
        c->chan.high_dyn = t->high_dyn;
        c->band.base = t->sig_dev;
        c->band.mask = ~0ULL;
        c->band.first_index = 0;
        c->band.limit = static_cast<unsigned long long>(t->max_len) + 2ULL;
        c->band.fmt = kCf32;
        c->item.channel = 0;
        c->item.n = n;
        c->item.sample_index = 0;
        c->item.rem_carrier_phase_rad = rem_carrier_phase_in_rad;
        c->item.phase_step_rad = phase_step_rad;
        c->item.phase_rate_step_rad = phase_rate_step_rad;
        c->item.rem_code_phase_chips = rem_code_phase_chips;
        c->item.code_phase_step_chips = code_phase_step_chips;
        c->item.code_phase_rate_step_chips = code_phase_rate_step_chips;
        int slices = (n + 4 * kTrkTile - 1) / (4 * kTrkTile);
        if (slices < 1) slices = 1;
        if (slices > t->slices_cap) slices = t->slices_cap;
        uint64_t launched = 0;
        int rc = launch_trk_batch(&c->item, 1, &c->chan, &c->band, c->out, B200_MAX_TAPS, slices, t->partial, t->counter,
            c->chan.code_len, 1u << t->taps, 1u << kCf32, t->stream, launched);
        if (rc) return rc;
        t->e->launches += launched;
        B200_CUDA_TRY(cudaStreamSynchronize(t->stream));
        for (int k = 0; k < t->taps; k++)
            {
                corr_out_host[k].re = c->out[k].x;
                corr_out_host[k].im = c->out[k].y;
            }
        return B200_OK;
    }

    // ---- Cpu_Multicorrelator (complex local code), cpu_multicorrelator.cc:53-100 --------------------------------------
    int b200_trk_set_local_code_and_taps_cplx(b200_trk* t, int code_length_chips, const b200_cf32* local_code_in, const float* shifts_chips)
    {
        if (!t || !local_code_in || !shifts_chips || code_length_chips < 1) return B200_ERR_ARG;
        B200_ENTER_DEVICE(t->e->device);
        // the code table last: b200_trk_correlate_cplx takes a code table to mean that the output buffer exists
        if (!t->out_cplx_dev) B200_CUDA_TRY(t->out_cplx_dev.alloc(B200_MAX_TAPS));
        if (const int rc = load_code(t, t->cplx_code_dev, local_code_in, code_length_chips)) return rc;
        t->cplx_code_len = code_length_chips;
        for (int k = 0; k < t->taps; k++) t->var_shifts[k] = shifts_chips[k];
        return B200_OK;
    }

    int b200_trk_correlate_cplx(b200_trk* t, const b200_cf32* sig_in_host, float rem_carrier_phase_in_rad, float phase_step_rad,
        float rem_code_phase_chips, float code_phase_step_chips, int signal_length_samples, b200_cf32* corr_out_host)
    {
        if (!t || !sig_in_host || !corr_out_host) return B200_ERR_ARG;
        if (!t->cplx_code_dev)
            {
                set_error("correlate before set_local_code_and_taps_cplx");
                return B200_ERR_STATE;
            }
        const int n = signal_length_samples;
        if (const int rc = stage_signal(t, t->sig_dev, sig_in_host, n, sizeof(float2))) return rc;
        uint64_t launched = 0;
        const int rc = launch_trk_cplx_code(t->sig_dev, t->cplx_code_dev, n, t->cplx_code_len, t->taps, t->var_shifts, rem_carrier_phase_in_rad,
            phase_step_rad, rem_code_phase_chips, code_phase_step_chips, t->out_cplx_dev, t->stream, launched);
        if (rc) return rc;
        t->e->launches += launched;
        B200_CUDA_TRY(cudaMemcpyAsync(corr_out_host, t->out_cplx_dev, sizeof(float2) * t->taps, cudaMemcpyDeviceToHost, t->stream));
        B200_CUDA_TRY(cudaStreamSynchronize(t->stream));
        return B200_OK;
    }

    // ---- Cpu_Multicorrelator_16sc (16-bit samples and code), cpu_multicorrelator_16sc.cc:47-91 -------------------------
    int b200_trk_set_local_code_and_taps_16sc(b200_trk* t, int code_length_chips, const int16_t* local_code_iq, const float* shifts_chips)
    {
        if (!t || !local_code_iq || !shifts_chips || code_length_chips < 1) return B200_ERR_ARG;
        B200_ENTER_DEVICE(t->e->device);
        // the code table last: b200_trk_correlate_16sc takes a code table to mean that all three buffers exist
        if (!t->sig16_dev) B200_CUDA_TRY(t->sig16_dev.alloc(2 * (static_cast<size_t>(t->max_len) + 2)));
        if (!t->out16_dev) B200_CUDA_TRY(t->out16_dev.alloc(2 * B200_MAX_TAPS));
        if (const int rc = load_code(t, t->code16_dev, local_code_iq, 2 * static_cast<size_t>(code_length_chips))) return rc;
        t->code16_len = code_length_chips;
        for (int k = 0; k < t->taps; k++) t->var_shifts[k] = shifts_chips[k];
        return B200_OK;
    }

    int b200_trk_correlate_16sc(b200_trk* t, const int16_t* sig_in_iq_host, float rem_carrier_phase_in_rad, float phase_step_rad,
        float rem_code_phase_chips, float code_phase_step_chips, int signal_length_samples, int16_t* corr_out_iq_host)
    {
        if (!t || !sig_in_iq_host || !corr_out_iq_host) return B200_ERR_ARG;
        if (!t->code16_dev)
            {
                set_error("correlate before set_local_code_and_taps_16sc");
                return B200_ERR_STATE;
            }
        const int n = signal_length_samples;
        if (const int rc = stage_signal(t, t->sig16_dev, sig_in_iq_host, n, 2 * sizeof(short))) return rc;
        uint64_t launched = 0;
        const int rc = launch_trk_16sc(t->sig16_dev, t->code16_dev, n, t->code16_len, t->taps, t->var_shifts, rem_carrier_phase_in_rad, phase_step_rad,
            rem_code_phase_chips, code_phase_step_chips, t->out16_dev, t->stream, launched);
        if (rc) return rc;
        t->e->launches += launched;
        B200_CUDA_TRY(cudaMemcpyAsync(corr_out_iq_host, t->out16_dev, sizeof(short) * 2 * t->taps, cudaMemcpyDeviceToHost, t->stream));
        B200_CUDA_TRY(cudaStreamSynchronize(t->stream));
        return B200_OK;
    }

    int b200_trk_destroy(b200_trk* t)
    {
        if (!t) return B200_ERR_ARG;
        cudaSetDevice(t->e->device);
        delete t;
        return B200_OK;
    }
}
