// TEST INFRASTRUCTURE ONLY.  The reference's pulse-blanking input filter (pulse_blanking_cc.cc, compiled where it lies by
// oracle/Makefile) driven over an in-memory stream the way GNU Radio's scheduler drives a general block: the input arrives
// in chunks, and each general_work call sees every item not yet consumed.  (gr::shim::Runner offers at most 64 output items
// per call, fewer than one segment of the default length, so the calls are made here.)
#include <gnuradio/block.h>
#include <gnuradio/io_signature.h>
#include <volk_gnsssdr/volk_gnsssdr_alloc.h>
#include <gnss_block_interface.h>
#include <cstdint>
#include <cstring>
#include <vector>
// the block keeps its threshold and state private; the tests compare them with the device's, so they are read directly
#define private public
#include "pulse_blanking_cc.h"
#undef private

extern "C"
{
    /* volk_gnsssdr::vector's allocator asks for it (the shim declares it; ref_kernels.c defines it for the other oracles) */
    size_t volk_gnsssdr_get_alignment(void) { return 32; }

    /* x: n interleaved complex floats; chunk_ends: ascending cumulative ends of the n_chunks input chunks (the last one n).
     * Writes the block's outputs to out (2 floats each) and their count to *n_out, its thres_ to *thres, and the state it
     * carries after the last call: state[0] = n_segments_, state[1] = last_filtered_, *est = noise_power_estimation_. */
    int ref_pulse_blanking(float pfa, int32_t length, int32_t segments_est, int32_t segments_reset, const float* x, uint64_t n,
        const uint64_t* chunk_ends, int n_chunks, float* out, uint64_t* n_out, float* thres, int64_t* state, float* est)
    {
        pulse_blanking_cc_sptr blk = make_pulse_blanking_cc(pfa, length, segments_est, segments_reset);
        uint64_t read = 0, written = 0;
        for (int c = 0; c < n_chunks; c++)
            {
                const uint64_t end = chunk_ends[c] < n ? chunk_ends[c] : n;
                if (end <= read) continue;
                const int avail = static_cast<int>(end - read);
                gr_vector_int ninput(1, avail);
                gr_vector_const_void_star in(1, x + 2 * read);
                gr_vector_void_star outv(1, out + 2 * written);
                const int produced = blk->general_work(avail, ninput, in, outv);
                const std::vector<int> consumed = blk->shim_take_consumed();
                const int c0 = consumed.empty() ? 0 : consumed[0];
                blk->shim_advance(0, static_cast<uint64_t>(c0));
                read += static_cast<uint64_t>(c0);
                written += static_cast<uint64_t>(produced);
            }
        *n_out = written;
        *thres = blk->thres_;
        state[0] = blk->n_segments_;
        state[1] = blk->last_filtered_ ? 1 : 0;
        *est = blk->noise_power_estimation_;
        return 0;
    }

    /* the block's thres_ alone */
    float ref_pulse_blanking_threshold(float pfa, int32_t length)
    {
        pulse_blanking_cc_sptr blk = make_pulse_blanking_cc(pfa, length, 0, 0);
        return blk->thres_;
    }
}
