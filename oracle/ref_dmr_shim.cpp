// C-ABI shim over the reference's DMR receive path, compiled UNMODIFIED from /root/reference (src/gr/gr_dmr_sink.cpp,
// src/DMR/dmrframe.cpp and the src/MMDVM FEC / LC files they use; oracle/ref_dmr.mk, run by build()), plus the lines of
// DMRControl::processAudio (src/DMR/dmrcontrol.cpp:225-271) that run the AMBE FEC and the EMB decode.
// TEST INFRASTRUCTURE ONLY (oracle/_ref/libqrl_ref_dmr.so): pins qrl_dmr.cu and tests/dmr_model.py to the reference's own code
// (tests/test_dmr_codec.py).  Nothing of the product links or loads this.  DMRFrame and gr_dmr_sink keep AT, LCSS, the downlink flag
// and the active slot private; the shim reads them by opening the access specifiers of those two headers for itself.
#include <cstring>
#include <vector>
#include <gnuradio/sync_block.h>     // the runtime stand-in and the standard headers, before the access specifiers open
#include <gnuradio/io_signature.h>
#define private public
#include "src/gr/gr_dmr_sink.h"
#undef private
#include "src/MMDVM/AMBEFEC.h"
#include "src/MMDVM/DMREMB.h"
#include "src/MMDVM/Golay2087.h"
#include "src/MMDVM/Golay24128.h"
#include "src/MMDVM/QR1676.h"
#include "src/MMDVM/CRC.h"

namespace {
struct Ref {
    DMRTiming timing;
    gr_dmr_sink sink{ &timing };
};

// one 72-byte record of qrl_dmr_rx (include/qrl_b200.h) from a frame the sink cut; position and ts_index filled by the caller
void record(DMRFrame& f, int ambe_fec, unsigned char* r)
{
    std::memset(r, 0, 72);
    r[9] = f.getFrameType(); r[10] = f.getFN(); r[11] = f._downlink; r[12] = f.cachDecoded(); r[13] = f._at; r[14] = f.getSlotNo();
    r[15] = f._lcss; r[16] = f.getColorCode(); r[17] = f.getDataType();
    r[18] = f.validate();
    int ambe = -1;
    if (f.getFrameType() != DMRFrameTypeData) {
        if (ambe_fec) ambe = f.runAudioFEC();
        if (f.getDataType() == DT_VOICE) {
            unsigned char d[33];
            f.getData(d);
            CDMREMB emb;
            emb.putData(d);
            r[21] = emb.getColorCode(); r[22] = emb.getPI(); r[23] = emb.getLCSS();
        }
    }
    r[19] = f.getFLCO(); r[20] = f.getFID();
    const uint32_t src = f.getSrcId(), dst = f.getDstId();
    std::memcpy(r + 24, &src, 4); std::memcpy(r + 28, &dst, 4); std::memcpy(r + 32, &ambe, 4);
    f.getCACH(r + 36);
    f.getData(r + 39);
}
}  // namespace

extern "C" {

void* ref_dmr_create() { return new Ref(); }
void ref_dmr_destroy(void* h) { delete static_cast<Ref*>(h); }

// gr_dmr_sink::work over `n` bits in calls of chunk[0], chunk[1], ... bits (cycled; a chunk of 1 gives exact positions and slots),
// then DMRFrame::validate and processAudio's FEC / EMB per frame.  Returns the number of records written (at most max_rec).
// With chunks longer than one bit, position and ts_index are those of the call's last bit.
int ref_dmr_work(void* hv, const unsigned char* bits, long n, const int* chunks, int n_chunks, int ambe_fec, unsigned char* out, int max_rec)
{
    Ref* h = static_cast<Ref*>(hv);
    int nrec = 0, k = 0;
    long p = 0;
    while (p < n) {
        long len = chunks[k++ % n_chunks];
        if (len > n - p) len = n - p;
        const int ts = h->sink._next_slot;
        gr_vector_const_void_star in{ bits + p };
        gr_vector_void_star o;
        h->sink.work(static_cast<int>(len), in, o);
        h->sink.stub_advance(len, 0);
        p += len;
        for (DMRFrame& f : h->sink.get_data()) {
            if (nrec < max_rec) {
                unsigned char* r = out + 72L * nrec;
                record(f, ambe_fec, r);
                const long long pos = p - 1;
                std::memcpy(r, &pos, 8);
                r[8] = static_cast<unsigned char>(ts);
            }
            nrec++;
        }
    }
    return nrec;
}

// the DMRTiming calls so far: increment_sample_counter count, and the slot numbers of set_slot_times in order
long ref_dmr_timing(void* hv, unsigned char* slots, int cap, int* n_slots)
{
    Ref* h = static_cast<Ref*>(hv);
    const int n = static_cast<int>(h->timing.slot_times.size());
    for (int i = 0; i < n && i < cap; i++) slots[i] = h->timing.slot_times[i];
    *n_slots = n;
    return static_cast<long>(h->timing.increments);
}

// the FEC building blocks, for exhaustive checks
int ref_golay2087_decode(uint32_t w20) { unsigned char b[3] = { (unsigned char)(w20 >> 12), (unsigned char)(w20 >> 4), (unsigned char)(w20 << 4) }; return CGolay2087::decode(b); }
int ref_qr1676_decode(uint32_t w16) { unsigned char b[2] = { (unsigned char)(w16 >> 8), (unsigned char)w16 }; return CQR1676::decode(b); }
int ref_golay24128_decode(uint32_t w24, uint32_t* out) { unsigned int o = 0; const bool v = CGolay24128::decode24128(w24, o); *out = o; return v; }
uint32_t ref_golay23127_decode(uint32_t w23) { return CGolay24128::decode23127(w23); }
uint32_t ref_golay24128_encode(uint32_t d) { return CGolay24128::encode24128(d); }
uint32_t ref_golay23127_encode(uint32_t d) { return CGolay24128::encode23127(d); }
int ref_crc_ccitt_check(const unsigned char* p12) { return CCRC::checkCCITT162(p12, 12U); }

}  // extern "C"
