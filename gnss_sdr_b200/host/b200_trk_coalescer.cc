/*!
 * \file b200_trk_coalescer.cc
 * \brief see header.
 */
#include "b200_trk_coalescer.h"
#include "b200_multicorrelator_real_codes.h"  // b200::shared_engine
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#if defined(__x86_64__) || defined(__i386__)
#include <immintrin.h>
#define B200_CPU_RELAX() _mm_pause()
#else
#define B200_CPU_RELAX() std::this_thread::yield()
#endif

namespace b200
{
Trk_Coalescer* Trk_Coalescer::instance()
{
    static std::mutex mu;
    static Trk_Coalescer* inst = nullptr;
    std::lock_guard<std::mutex> lk(mu);
    if (inst == nullptr)
        {
            b200_engine* eng = shared_engine();
            if (eng == nullptr) return nullptr;
            inst = new Trk_Coalescer(eng);  // lives as long as the process (block destructors may still call it at exit)
        }
    return inst;
}


Trk_Coalescer::Trk_Coalescer(b200_engine* engine) : d_engine(engine), d_slots(new Slot[kMaxChannels])
{
    for (auto& w : d_band_written) w.store(0);
    for (auto& w : d_band_lo) w.store(0);
    for (auto& w : d_band_active) w.store(0);
    for (auto& w : d_band_attached) w.store(0);
    if (const char* env = std::getenv("B200_COALESCE_WINDOW_US")) d_window_us = std::atoi(env);
    d_thread = std::thread([this] { tick_loop(); });
}


Trk_Coalescer::~Trk_Coalescer()
{
    d_stop.store(true);
    d_posted.fetch_add(1);  // wake the tick thread
    d_posted.notify_all();
    d_done_gen.fetch_add(1);
    d_done_gen.notify_all();
    for (int b = 0; b < kMaxBands; b++) d_cv_space[b].notify_all();
    if (d_thread.joinable()) d_thread.join();
}


bool Trk_Coalescer::ensure_band(int band, uint64_t capacity_samples)
{
    if (band < 0 || band >= kMaxBands) return false;
    std::lock_guard<std::mutex> lk(d_admin_mu);
    if (d_band_capacity[band] != 0) return true;
    if (capacity_samples == 0)
        {
            const char* env = std::getenv("B200_BAND_CAPACITY");
            capacity_samples = env ? std::strtoull(env, nullptr, 10) : (1ULL << 23);
        }
    uint64_t cap = 2;
    while (cap < capacity_samples) cap <<= 1;
    if (b200_iq_create(d_engine, band, cap) != B200_OK)
        {
            std::snprintf(d_error, sizeof(d_error), "%s", b200_last_error());
            return false;
        }
    d_band_capacity[band] = cap;
    return true;
}


Trk_Coalescer::Slot* Trk_Coalescer::slot_of(int id)
{
    if (id < 0 || id >= kMaxChannels || d_slots[id].state.load(std::memory_order_acquire) == FREE) return nullptr;
    return &d_slots[id];
}


int Trk_Coalescer::open_channel(int band, int n_correlators)
{
    if (!ensure_band(band)) return -1;
    int id = -1;
    if (b200_trk_channel_create(d_engine, band, n_correlators, &id) != B200_OK || id >= kMaxChannels)
        {
            std::snprintf(d_error, sizeof(d_error), "%s", id >= kMaxChannels ? "more than 4096 channels" : b200_last_error());
            return -1;
        }
    std::lock_guard<std::mutex> lk(d_admin_mu);
    Slot& s = d_slots[id];
    s.band = band;
    s.taps = n_correlators;
    s.active.store(false);
    s.attached.store(false);
    s.cursor.store(0);
    s.state.store(IDLE, std::memory_order_release);
    if (id + 1 > d_n_slots.load()) d_n_slots.store(id + 1);
    return id;
}


// A channel starts (or resumes) offering samples.  When no other channel is attached to its band, nothing says that the
// stream it is in continues the one the band last saw (a flowgraph restarted in the same process starts its sample counter
// over): what the band holds is forgotten, and the channel's own push refills it.  "Attached" lasts from a channel's first
// push to its idle() / close_channel(); missing a batch window only makes a channel inactive, it keeps its claim on the band
// (it may be between push and post).
void Trk_Coalescer::activate(Slot& s, bool stream_may_be_new)
{
    std::lock_guard<std::mutex> lk(d_band_mu[s.band]);
    if (!s.active.exchange(true))
        {
            d_n_active.fetch_add(1);
            d_band_active[s.band].fetch_add(1);
        }
    if (!s.attached.exchange(true))
        {
            if (d_band_attached[s.band].fetch_add(1) == 0 && stream_may_be_new)
                {
                    d_band_written[s.band].store(0, std::memory_order_release);
                    d_band_lo[s.band].store(0, std::memory_order_release);
                    b200_iq_forget(d_engine, s.band);
                }
        }
}


void Trk_Coalescer::deactivate(Slot& s)
{
    if (s.active.exchange(false))
        {
            d_n_active.fetch_sub(1);
            d_band_active[s.band].fetch_sub(1);
        }
}


void Trk_Coalescer::idle(int id)
{
    Slot* s = slot_of(id);
    if (s == nullptr) return;
    deactivate(*s);
    if (s->attached.exchange(false)) d_band_attached[s->band].fetch_sub(1);
    d_cv_space[s->band].notify_all();
    d_posted.notify_all();  // the tick thread re-evaluates how many posts it is waiting for
}


void Trk_Coalescer::close_channel(int id)
{
    Slot* s = slot_of(id);
    if (s == nullptr) return;
    // an epoch still in flight finishes first (its result is dropped)
    for (;;)
        {
            const uint32_t gen = d_done_gen.load(std::memory_order_acquire);
            const int st = s->state.load(std::memory_order_acquire);
            if (st != POSTED && st != IN_FLIGHT) break;
            if (d_stop.load()) break;
            d_done_gen.wait(gen, std::memory_order_acquire);
        }
    idle(id);
    s->state.store(IDLE);  // engine channel ids are never reused; the slot just goes quiet
}


bool Trk_Coalescer::set_code(int id, int code_length_chips, const float* code, const float* shifts_chips, bool high_dynamics)
{
    if (slot_of(id) == nullptr) return false;
    return b200_trk_channel_set_code(d_engine, id, code_length_chips, code, shifts_chips, high_dynamics ? 1 : 0) == B200_OK;
}


bool Trk_Coalescer::set_taps(int id, const float* shifts_chips)
{
    return b200_trk_channel_set_taps(d_engine, id, shifts_chips) == B200_OK;
}


// would [abs_index, abs_index + n) still leave the oldest sample an active channel of this band needs in the ring?
bool Trk_Coalescer::fits(int band, uint64_t abs_index, uint64_t n) const
{
    const uint64_t cap = d_band_capacity[band];
    uint64_t oldest = abs_index;
    const int ns = d_n_slots.load(std::memory_order_acquire);
    for (int i = 0; i < ns; i++)
        {
            const Slot& o = d_slots[i];
            if (o.band == band && o.active.load(std::memory_order_relaxed))
                {
                    const uint64_t c = o.cursor.load(std::memory_order_relaxed);
                    if (c < oldest) oldest = c;
                }
        }
    return abs_index + n - oldest <= cap - cap / 8;
}


bool Trk_Coalescer::push(int id, uint64_t abs_index, const std::complex<float>* samples, uint64_t n, bool* behind)
{
    if (behind) *behind = false;
    Slot* s = slot_of(id);
    if (s == nullptr) return false;
    const int band = s->band;
    s->cursor.store(abs_index, std::memory_order_relaxed);
    if (!s->active.load(std::memory_order_acquire)) activate(*s, true);
    d_samples_offered.fetch_add(n, std::memory_order_relaxed);
    // fast path: somebody has already put these samples into the band (every block of the flowgraph offers the same stream)
    if (abs_index >= d_band_lo[band].load(std::memory_order_acquire) && abs_index + n <= d_band_written[band].load(std::memory_order_acquire)) return true;

    // One producer at a time.  The others do not queue on the mutex (32 hand-overs of a contended lock cost more than the
    // copy itself): whoever gets it copies, the rest watch the band's written range, which usually comes to cover them.
    std::unique_lock<std::mutex> lk(d_band_mu[band], std::try_to_lock);
    for (int spins = 0; !lk.owns_lock(); spins++)
        {
            if (abs_index >= d_band_lo[band].load(std::memory_order_acquire) && abs_index + n <= d_band_written[band].load(std::memory_order_acquire)) return true;
            if (d_stop.load(std::memory_order_relaxed)) return false;
            if (spins < 64)
                B200_CPU_RELAX();
            else
                std::this_thread::yield();
            if ((spins & 7) == 7) (void)lk.try_lock();
        }
    if (abs_index >= d_band_lo[band].load(std::memory_order_acquire) && abs_index + n <= d_band_written[band].load(std::memory_order_acquire)) return true;
    if (d_band_attached[band].load(std::memory_order_acquire) > 1 && d_band_written[band].load() > d_band_lo[band].load())
        {
            // the band is shared right now: its window may only grow at the top
            if (abs_index < d_band_lo[band].load())
                {
                    std::snprintf(d_error, sizeof(d_error), "channel %d is behind the band's window (sample %llu < %llu)", id,
                        static_cast<unsigned long long>(abs_index), static_cast<unsigned long long>(d_band_lo[band].load()));
                    if (behind) *behind = true;
                    return false;
                }
            // ahead of everything pushed so far: the channels behind are about to offer the samples in between - give them a
            // moment (the lock is released while waiting); if they do not, the band restarts here and THEY take the path above
            if (abs_index > d_band_written[band].load())
                d_cv_space[band].wait_for(lk, std::chrono::milliseconds(20),
                    [&] { return d_stop.load() || abs_index <= d_band_written[band].load() || d_band_attached[band].load() <= 1; });
            if (abs_index >= d_band_lo[band].load() && abs_index + n <= d_band_written[band].load()) return true;
        }
    // back-pressure: never overwrite what a slower active channel of this band still needs.  A channel that stopped calling
    // (stalled test thread, block torn down without idle()) must not wedge the rest: after the timeout laggards go idle.
    if (!fits(band, abs_index, n))
        {
            if (!d_cv_space[band].wait_for(lk, std::chrono::milliseconds(2000), [&] { return d_stop.load() || fits(band, abs_index, n); }))
                {
                    const uint64_t cap = d_band_capacity[band];
                    const int ns = d_n_slots.load();
                    for (int i = 0; i < ns; i++)
                        {
                            Slot& o = d_slots[i];
                            if (o.band == band && o.active.load() && abs_index + n - o.cursor.load() > cap - cap / 8) deactivate(o);
                        }
                }
        }
    uint64_t n_new = 0;
    const int rc = b200_iq_push_at(d_engine, band, abs_index, reinterpret_cast<const b200_cf32*>(samples), n, &n_new);
    if (rc != B200_OK)
        {
            std::snprintf(d_error, sizeof(d_error), "%s", b200_last_error());
            return false;
        }
    d_samples_copied.fetch_add(n_new, std::memory_order_relaxed);
    // the band's window after this push (a gap or a stream that started over moves its lower edge)
    uint64_t lo = 0, hi = 0;
    if (b200_iq_window(d_engine, band, &lo, &hi) == B200_OK)
        {
            // order matters for the lock-free fast path: shrink first (lo up / hi down), then grow
            d_band_written[band].store(std::min<uint64_t>(hi, d_band_written[band].load(std::memory_order_relaxed)), std::memory_order_release);
            d_band_lo[band].store(lo, std::memory_order_release);
            d_band_written[band].store(hi, std::memory_order_release);
        }
    d_cv_space[band].notify_all();  // a channel ahead of the band may be waiting for this range
    return true;
}


bool Trk_Coalescer::post(int id, uint64_t abs_index, int n, float rem_carrier_phase_rad, float phase_step_rad, float phase_rate_step_rad,
    float rem_code_phase_chips, float code_phase_step_chips, float code_phase_rate_step_chips)
{
    Slot* s = slot_of(id);
    if (s == nullptr) return false;
    const int st = s->state.load(std::memory_order_acquire);
    if (st == POSTED || st == IN_FLIGHT) return false;
    s->item.channel = id;
    s->item.n = n;
    s->item.sample_index = abs_index;
    s->item.rem_carrier_phase_rad = rem_carrier_phase_rad;
    s->item.phase_step_rad = phase_step_rad;
    s->item.phase_rate_step_rad = phase_rate_step_rad;
    s->item.rem_code_phase_chips = rem_code_phase_chips;
    s->item.code_phase_step_chips = code_phase_step_chips;
    s->item.code_phase_rate_step_chips = code_phase_rate_step_chips;
    s->cursor.store(abs_index, std::memory_order_relaxed);
    if (!s->active.load(std::memory_order_acquire)) activate(*s, false);
    s->t_post = std::chrono::steady_clock::now();
    s->state.store(POSTED, std::memory_order_release);
    // a slower channel may have been waiting for this cursor to move
    d_cv_space[s->band].notify_all();
    if (d_posted.fetch_add(1, std::memory_order_acq_rel) == 0) d_posted.notify_one();
    return true;
}


bool Trk_Coalescer::wait(int id, std::complex<float>* out)
{
    Slot* s = slot_of(id);
    if (s == nullptr) return false;
    // spin briefly (the GPU round trip of a batch is tens of microseconds), then sleep on the slot's state word - but only
    // while the block threads leave cores free: with more waiters than half the hardware threads, spinning waiters push the
    // tick thread off its core and the batch round trip grows several-fold
    static const int hw = static_cast<int>(std::thread::hardware_concurrency());
    const int spin_limit = (d_n_active.load(std::memory_order_relaxed) * 2 <= hw) ? 2000 : 0;
    int st;
    int spins = 0;
    for (;;)
        {
            // generation first: a batch that completes between the two loads changes it and the wait below returns at once
            const uint32_t gen = d_done_gen.load(std::memory_order_acquire);
            st = s->state.load(std::memory_order_acquire);
            if (st != POSTED && st != IN_FLIGHT) break;
            if (d_stop.load(std::memory_order_relaxed)) return false;
            if (++spins < spin_limit)
                {
                    B200_CPU_RELAX();
                    continue;
                }
            d_done_gen.wait(gen, std::memory_order_acquire);
        }
    const bool ok = st == DONE;
    if (ok)
        {
            for (int k = 0; k < s->taps; k++) out[k] = s->out[k];
            const double us = std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - s->t_post).count();
            s->lat_sum_us += us;   // per slot: 256 threads woken together must not queue on one mutex for a statistic
            s->lat_max_us = std::max(s->lat_max_us, us);
        }
    if (st == DONE || st == FAILED) s->state.store(IDLE, std::memory_order_release);
    return ok;
}


void Trk_Coalescer::tick_loop()
{
    std::vector<b200_trk_item> items;
    std::vector<int> ids;
    std::vector<b200_cf32> taps;
    while (!d_stop.load(std::memory_order_acquire))
        {
            // sleep until somebody posts
            while (d_posted.load(std::memory_order_acquire) == 0 && !d_stop.load()) d_posted.wait(0, std::memory_order_acquire);
            if (d_stop.load()) break;
            // every active channel is expected to post; stragglers get d_window_us from the first post seen
            const auto deadline = std::chrono::steady_clock::now() + std::chrono::microseconds(d_window_us);
            bool expired = false;
            while (d_posted.load(std::memory_order_acquire) < d_n_active.load(std::memory_order_acquire))
                {
                    if (std::chrono::steady_clock::now() >= deadline)
                        {
                            expired = true;
                            break;
                        }
                    B200_CPU_RELAX();
                }
            items.clear();
            ids.clear();
            const int ns = d_n_slots.load(std::memory_order_acquire);
            for (int i = 0; i < ns; i++)
                {
                    Slot& s = d_slots[i];
                    int want = POSTED;
                    if (s.state.load(std::memory_order_acquire) == POSTED && s.state.compare_exchange_strong(want, IN_FLIGHT))
                        {
                            items.push_back(s.item);
                            ids.push_back(i);
                        }
                }
            d_posted.fetch_sub(static_cast<int>(items.size()), std::memory_order_acq_rel);
            if (items.empty()) continue;
            if (expired)
                {
                    // who did not make it is not waited for next time (posting makes it active again)
                    for (int i = 0; i < ns; i++)
                        {
                            Slot& s = d_slots[i];
                            const int st = s.state.load();
                            if (s.active.load() && st != IN_FLIGHT && st != POSTED) deactivate(s);
                        }
                }
            const auto t0 = std::chrono::steady_clock::now();
            taps.resize(items.size() * B200_MAX_TAPS);
            uint64_t ticket = 0;
            int rc = b200_trk_submit(d_engine, items.data(), static_cast<int>(items.size()), B200_MAX_TAPS, &ticket);
            if (rc == B200_OK) rc = b200_trk_wait(d_engine, ticket, taps.data());
            const double us = std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t0).count();
            if (rc != B200_OK) std::snprintf(d_error, sizeof(d_error), "%s", b200_last_error());
            for (size_t k = 0; k < ids.size(); k++)
                {
                    Slot& s = d_slots[ids[k]];
                    if (rc == B200_OK)
                        for (int t = 0; t < s.taps; t++) s.out[t] = std::complex<float>(taps[k * B200_MAX_TAPS + t].re, taps[k * B200_MAX_TAPS + t].im);
                    s.state.store(rc == B200_OK ? DONE : FAILED, std::memory_order_release);
                }
            // ONE wake call for the whole batch: all waiters sleep on the generation word (a futex wake per slot costs the
            // tick thread ~2 us each - with 256 channels that was most of the time between batches)
            d_done_gen.fetch_add(1, std::memory_order_release);
            d_done_gen.notify_all();
            {
                std::lock_guard<std::mutex> lk(d_admin_mu);
                d_stats.batches++;
                d_stats.items += items.size();
                d_stats.sum_batch_us += us;
                if (expired) d_stats.window_expired++;
            }
        }
}


Trk_Coalescer::Stats Trk_Coalescer::stats()
{
    std::lock_guard<std::mutex> lk(d_admin_mu);
    Stats s = d_stats;
    const int ns = d_n_slots.load();
    for (int i = 0; i < ns; i++)
        {
            s.sum_latency_us += d_slots[i].lat_sum_us;
            s.max_latency_us = std::max(s.max_latency_us, d_slots[i].lat_max_us);
        }
    s.samples_copied = d_samples_copied.load();
    s.samples_offered = d_samples_offered.load();
    return s;
}


void Trk_Coalescer::reset_stats()
{
    std::lock_guard<std::mutex> lk(d_admin_mu);
    d_stats = Stats();
    const int ns = d_n_slots.load();
    for (int i = 0; i < ns; i++) d_slots[i].lat_sum_us = d_slots[i].lat_max_us = 0.0;
    d_samples_copied.store(0);
    d_samples_offered.store(0);
}
}  // namespace b200
