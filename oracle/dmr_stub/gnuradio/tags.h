// oracle/gr_stub/gnuradio/tags.h plus the two pmt calls gr_dmr_sink.cpp makes on rx_time tags (tuple_ref, to_double).  The shim
// places no tags, so they are never reached.  TEST INFRASTRUCTURE ONLY (oracle/ref_dmr.mk).
#pragma once
#include_next <gnuradio/tags.h>
namespace pmt {
inline pmt_t tuple_ref(const pmt_t& p, size_t) { return p; }
inline double to_double(const pmt_t& p) { return p->f32; }
}  // namespace pmt
