// TEST INFRASTRUCTURE ONLY.  The reference's notch input filters (notch_cc.cc and notch_lite_cc.cc, compiled where they lie
// by oracle/notch.mk) driven over an in-memory stream the way GNU Radio's scheduler drives them: the input arrives in chunks
// and each general_work call sees every item not yet consumed.  NotchLite has set_history(2), so each call's input starts
// with one history item: a zero ahead of sample 0, then the last consumed sample.  Notch has no history.
#include <gnuradio/block.h>
#include <gnuradio/io_signature.h>
#include <volk_gnsssdr/volk_gnsssdr_alloc.h>
#include <gnss_block_interface.h>
#include <complex>
#include <cstdint>
#include <cstring>
#include <vector>
// the blocks keep their state private; the tests compare it with the device's, so it is read directly
#define private public
#include "notch_cc.h"
#include "notch_lite_cc.h"
#undef private

namespace
{
// one general_work call of blk over x[read, end) (Lite: with its history item); returns the items consumed
template <typename B>
int call(B& blk, bool lite, const float* x, uint64_t read, uint64_t end, float* out)
{
    const int avail = static_cast<int>(end - read);
    std::vector<std::complex<float>> buf;
    const void* in_ptr = x + 2 * read;
    if (lite)
        {
            buf.resize(static_cast<size_t>(avail) + 1);
            buf[0] = read == 0 ? std::complex<float>(0.f, 0.f) : std::complex<float>(x[2 * read - 2], x[2 * read - 1]);
            std::memcpy(static_cast<void*>(buf.data() + 1), x + 2 * read, sizeof(float) * 2 * static_cast<size_t>(avail));
            in_ptr = buf.data();
        }
    gr_vector_int ninput(1, avail + (lite ? 1 : 0));
    gr_vector_const_void_star in(1, in_ptr);
    gr_vector_void_star outv(1, out);
    blk.general_work(avail, ninput, in, outv);
    const std::vector<int> consumed = blk.shim_take_consumed();
    const int c0 = consumed.empty() ? 0 : consumed[0];
    blk.shim_advance(0, static_cast<uint64_t>(c0));
    return c0;
}

template <typename B>
void fill_state(const B& blk, int64_t* state, float* f)
{
    state[0] = blk.n_segments_;
    state[1] = blk.filter_state_ ? 1 : 0;
    f[0] = blk.noise_pow_est_;
    f[1] = blk.thres_;
    f[2] = blk.z_0_.real();
    f[3] = blk.z_0_.imag();
    f[4] = blk.last_out_.real();
    f[5] = blk.last_out_.imag();
}
}  // namespace

extern "C"
{
    /* volk_gnsssdr::vector's allocator asks for it (the shim declares it; ref_kernels.c defines it for the other oracles) */
    size_t volk_gnsssdr_get_alignment(void) { return 32; }

    /* variant 0 Notch, 1 NotchLite.  x: n interleaved complex floats; chunk_ends: ascending cumulative ends of the n_chunks
     * input chunks.  Writes the outputs to out (2 floats each) and their count to *n_out; state = {n_segments_,
     * filter_state_, n_segments_coeff_ (Lite)}, f = {noise_pow_est_, thres_, z_0_, last_out_} after the last call.
     * per_segment != 0: the stream is fed one segment per call instead (chunk_ends is not read), and after segment k
     * est[k] = noise_pow_est_, and z0[2 (k L + i)] the z0 sample i used (Lite: z_0_; Notch: exp(i angle_[i]) as the block
     * forms it); both are only meaningful where the segment used them. */
    int ref_notch(int variant, float pfa, float p_c_factor, int32_t length, int32_t segments_est, int32_t segments_reset, int32_t segments_coeff,
        const float* x, uint64_t n, const uint64_t* chunk_ends, int n_chunks, int per_segment, float* out, uint64_t* n_out, int64_t* state,
        float* f, float* est, float* z0)
    {
        const bool lite = variant == 1;
        notch_sptr nb;
        notch_lite_sptr lb;
        if (lite)
            lb = make_notch_filter_lite(p_c_factor, pfa, length, segments_est, segments_reset, segments_coeff);
        else
            nb = make_notch_filter(pfa, p_c_factor, length, segments_est, segments_reset);
        uint64_t read = 0, written = 0;
        const uint64_t L = static_cast<uint64_t>(length);
        if (per_segment)
            {
                for (uint64_t k = 0; read + L + 1 <= n; k++)
                    {
                        const int c = lite ? call(*lb, true, x, read, read + L + 1, out + 2 * written) : call(*nb, false, x, read, read + L + 1, out + 2 * written);
                        if (c == 0) break;
                        read += static_cast<uint64_t>(c);
                        written += static_cast<uint64_t>(c);
                        est[k] = lite ? lb->noise_pow_est_ : nb->noise_pow_est_;
                        for (uint64_t i = 0; i < L; i++)
                            {
                                std::complex<float> z = lite ? lb->z_0_ : std::exp(gr_complex(0.0, 1.0) * (*(nb->angle_.data() + i)));
                                z0[2 * (k * L + i)] = z.real();
                                z0[2 * (k * L + i) + 1] = z.imag();
                            }
                    }
            }
        else
            for (int c = 0; c < n_chunks; c++)
                {
                    const uint64_t end = chunk_ends[c] < n ? chunk_ends[c] : n;
                    if (end <= read) continue;
                    const int k = lite ? call(*lb, true, x, read, end, out + 2 * written) : call(*nb, false, x, read, end, out + 2 * written);
                    read += static_cast<uint64_t>(k);
                    written += static_cast<uint64_t>(k);
                }
        *n_out = written;
        if (lite)
            {
                fill_state(*lb, state, f);
                state[2] = lb->n_segments_coeff_;
            }
        else
            {
                fill_state(*nb, state, f);
                state[2] = 0;
            }
        return 0;
    }
}
