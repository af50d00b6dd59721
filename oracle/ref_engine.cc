/*
 * TEST INFRASTRUCTURE ONLY (oracle/) -- builds into oracle/_ref/liboracle_ref.so.
 *
 * extern "C" handle API around the reference's OWN class
 * Cpu_Multicorrelator_Real_Codes (src/algorithms/tracking/libs/
 * cpu_multicorrelator_real_codes.{h,cc}), whose .cc is compiled where it lies
 * under /root/reference by oracle/Makefile and linked here unmodified.
 *
 * Also the CPU-baseline timing harness, shaped like the reference's own
 * cpu_multicorrelator_real_codes_test.cc:41-62,135-169: T std::threads, each
 * owning one correlator object, each running `iters` back-to-back calls.
 */
#include "cpu_multicorrelator_real_codes.h"
#include <volk_gnsssdr/volk_gnsssdr.h>
#include <atomic>
#include <chrono>
#include <pthread.h>
#include <sched.h>
#include <complex>
#include <cstring>
#include <random>
#include <thread>
#include <vector>

namespace
{
struct RefMc
{
    Cpu_Multicorrelator_Real_Codes mc;
    float* code{nullptr};
    float* shifts{nullptr};
    std::complex<float>* out{nullptr};
    std::complex<float>* in{nullptr};
    int max_len{0};
    int taps{0};
    int code_len{0};
};
}  // namespace

extern "C"
{
    void* ref_mc_create(int max_len, int taps, int high_dyn)
    {
        auto* h = new RefMc();
        h->max_len = max_len;
        h->taps = taps;
        h->mc.init(max_len, taps);
        h->mc.set_high_dynamics_resampler(high_dyn != 0);
        h->shifts = static_cast<float*>(volk_gnsssdr_malloc(taps * sizeof(float), 32));
        h->out = static_cast<std::complex<float>*>(volk_gnsssdr_malloc(taps * sizeof(std::complex<float>), 32));
        h->in = static_cast<std::complex<float>*>(volk_gnsssdr_malloc((max_len + 16) * sizeof(std::complex<float>), 32));
        return h;
    }

    int ref_mc_set_code(void* hv, const float* code, int code_len, const float* shifts)
    {
        auto* h = static_cast<RefMc*>(hv);
        if (h->code) volk_gnsssdr_free(h->code);
        h->code = static_cast<float*>(volk_gnsssdr_malloc(code_len * sizeof(float), 32));
        std::memcpy(h->code, code, code_len * sizeof(float));
        std::memcpy(h->shifts, shifts, h->taps * sizeof(float));
        h->code_len = code_len;
        h->mc.set_local_code_and_taps(code_len, h->code, h->shifts);
        return 0;
    }

    /* One epoch: exactly do_correlation_step's call (dll_pll_veml_tracking.cc:1232-1245). */
    int ref_mc_correlate(void* hv, const float* in_iq, float rem_carr_rad, float phase_step_rad, float phase_rate_step_rad,
        float rem_code_chips, float code_step_chips, float code_rate_step_chips, int n, float* out_taps)
    {
        auto* h = static_cast<RefMc*>(hv);
        if (n > h->max_len) return -1;
        std::memcpy(h->in, in_iq, sizeof(std::complex<float>) * n);
        h->mc.set_input_output_vectors(h->out, h->in);
        h->mc.Carrier_wipeoff_multicorrelator_resampler(rem_carr_rad, phase_step_rad, phase_rate_step_rad,
            rem_code_chips, code_step_chips, code_rate_step_chips, n);
        std::memcpy(out_taps, h->out, sizeof(std::complex<float>) * h->taps);
        return 0;
    }

    /* The shifts array the reference object keeps a POINTER to (cpu_multicorrelator_real_codes.cc:53-63): tests mutate it in
     * place between correlations, as dll_pll_veml_tracking does (:1045-1053, :2132-2146). */
    float* ref_mc_shifts(void* hv) { return static_cast<RefMc*>(hv)->shifts; }

    void ref_mc_destroy(void* hv)
    {
        auto* h = static_cast<RefMc*>(hv);
        h->mc.free();
        if (h->code) volk_gnsssdr_free(h->code);
        volk_gnsssdr_free(h->shifts);
        volk_gnsssdr_free(h->out);
        volk_gnsssdr_free(h->in);
        delete h;
    }

    /*
     * CPU baseline timing.  `threads` correlators run concurrently; every call
     * correlates `n` samples x `taps` taps with a code of `code_len` values.
     * Each thread walks over `n_epochs_buf` distinct epochs of its own IQ buffer
     * (so the data is not pinned in L1), `iters` calls in total.
     * Returns elapsed wall seconds; channel-samples processed = threads*iters*n.
     */
    double ref_mc_bench_pinned(int threads, int n, int taps, int code_len, int iters, int n_epochs_buf, int high_dyn, int pin);
    double ref_mc_bench(int threads, int n, int taps, int code_len, int iters, int n_epochs_buf, int high_dyn)
    {
        return ref_mc_bench_pinned(threads, n, taps, code_len, iters, n_epochs_buf, high_dyn, 1);
    }

    /* pin != 0: thread t is bound to the t-th CPU of the process's affinity mask (round robin), so that the figure does
     * not depend on where the scheduler happens to put the threads. */
    double ref_mc_bench_pinned(int threads, int n, int taps, int code_len, int iters, int n_epochs_buf, int high_dyn, int pin)
    {
        std::vector<RefMc*> pool(threads);
        std::vector<std::vector<std::complex<float>>> iq(threads);
        std::vector<float> code(code_len);
        std::vector<float> shifts(taps);
        std::mt19937 rng(12345);
        std::uniform_real_distribution<float> ud(-1.0F, 1.0F);
        for (auto& c : code) c = (rng() & 1U) ? 1.0F : -1.0F;
        for (int t = 0; t < taps; t++) shifts[t] = (static_cast<float>(t) - static_cast<float>(taps - 1) / 2.0F) * 0.5F;
        for (int t = 0; t < threads; t++)
            {
                pool[t] = static_cast<RefMc*>(ref_mc_create(n, taps, high_dyn));
                ref_mc_set_code(pool[t], code.data(), code_len, shifts.data());
                iq[t].resize(static_cast<size_t>(n) * n_epochs_buf + 16);
                for (auto& v : iq[t]) v = std::complex<float>(ud(rng), ud(rng));
            }
        const float step = static_cast<float>(code_len) / static_cast<float>(n);
        auto worker = [&](int t) {
            RefMc* h = pool[t];
            for (int k = 0; k < iters; k++)
                {
                    const std::complex<float>* in = iq[t].data() + static_cast<size_t>(k % n_epochs_buf) * n;
                    h->mc.set_input_output_vectors(h->out, in);
                    h->mc.Carrier_wipeoff_multicorrelator_resampler(0.4F, 0.001F, 0.0F, 0.3F, step, 0.0F, n);
                }
        };
        std::vector<int> cpus;
        {
            cpu_set_t set;
            CPU_ZERO(&set);
            if (sched_getaffinity(0, sizeof(set), &set) == 0)
                for (int c = 0; c < CPU_SETSIZE; c++)
                    if (CPU_ISSET(c, &set)) cpus.push_back(c);
        }
        // all threads start together: the timed region is max over threads of the same amount of work
        std::atomic<int> ready{0};
        std::atomic<bool> go{false};
        auto gated = [&](int t) {
            if (pin && !cpus.empty())
                {
                    cpu_set_t one;
                    CPU_ZERO(&one);
                    CPU_SET(cpus[t % cpus.size()], &one);
                    pthread_setaffinity_np(pthread_self(), sizeof(one), &one);
                }
            // first touch of the thread's buffer from its own CPU (NUMA-local pages)
            volatile float sink = 0.f;
            for (size_t i = 0; i < iq[t].size(); i += 512) sink = sink + iq[t][i].real();
            ready++;
            while (!go.load(std::memory_order_acquire)) std::this_thread::yield();
            worker(t);
        };
        std::vector<std::thread> th;
        for (int t = 0; t < threads; t++) th.emplace_back(gated, t);
        while (ready.load() < threads) std::this_thread::yield();
        const auto t0 = std::chrono::steady_clock::now();
        go.store(true, std::memory_order_release);
        for (auto& x : th) x.join();
        const auto t1 = std::chrono::steady_clock::now();
        for (int t = 0; t < threads; t++) ref_mc_destroy(pool[t]);
        return std::chrono::duration<double>(t1 - t0).count();
    }
}
