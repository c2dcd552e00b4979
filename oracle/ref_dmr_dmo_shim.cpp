// C-ABI shim over the reference's DMR direct-mode receive path, compiled UNMODIFIED from the reference tree (src/gr/gr_dmr_dmo_sink.cpp,
// src/MMDVM/DMRSlotType2.cpp, src/DMR/dmrframe.cpp and the src/MMDVM FEC / LC files they use; oracle/ref_dmr_dmo.mk, run by build()),
// plus the lines of DMRControl::processAudio that run the AMBE FEC and the EMB decode, as ref_dmr_shim.cpp does.
// TEST INFRASTRUCTURE ONLY (oracle/_ref/libqrl_ref_dmr_dmo.so): pins qrl_dmr.cu's DMO sink and tests/dmr_dmo_model.py to the
// reference's own code (tests/test_dmr_dmo_codec.py).  Nothing of the product links or loads this.  The sink's constructor leaves
// m_bitBuffer, m_buffer, m_centre, m_threshold and m_control uninitialised; the shim sets them to zero after construction, which is the
// definition qrl_b200.h gives.  The sink's and the slot-type decoder's members are private; the shim opens the access specifiers of
// their headers for itself.
#include <cstring>
#include <vector>
#include <gnuradio/block.h>          // the runtime stand-in and the standard headers, before the access specifiers open
#include <gnuradio/io_signature.h>
#define private public
#include "src/gr/gr_dmr_dmo_sink.h"
#undef private
#include "src/MMDVM/DMREMB.h"

namespace {
struct Ref {
    gr_dmr_dmo_sink sink;
    long long pos = 0;           // samples processed since create
    Ref()
    {
        std::memset(sink.m_bitBuffer, 0, sizeof sink.m_bitBuffer);
        std::memset(sink.m_buffer, 0, sizeof sink.m_buffer);
        for (int i = 0; i < 4; i++) { sink.m_centre[i] = 0.0f; sink.m_threshold[i] = 0.0f; }
        sink.m_control = 0;
    }
};

// one 72-byte record of qrl_dmr_dmo_rx (include/qrl_b200.h) from a frame the sink wrote; position filled by the caller
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

void* ref_dmo_create() { return new Ref(); }
void ref_dmo_destroy(void* h) { delete static_cast<Ref*>(h); }

// gr_dmr_dmo_sink::processSample over n samples, one at a time (what general_work does), then DMRFrame::validate and processAudio's
// FEC / EMB per frame.  A record's position is the index, counted from create, of the sample whose processing wrote the frame.
// Returns the number of frames written (at most max_rec records are stored).
int ref_dmo_work(void* hv, const float* x, long n, int ambe_fec, unsigned char* out, int max_rec)
{
    Ref* h = static_cast<Ref*>(hv);
    int nrec = 0;
    for (long i = 0; i < n; i++, h->pos++) {
        h->sink.processSample(x[i]);
        if (h->sink._frame_buffer.empty()) continue;
        for (DMRFrame& f : h->sink.get_data()) {
            if (nrec < max_rec) {
                unsigned char* r = out + 72L * nrec;
                record(f, ambe_fec, r);
                std::memcpy(r, &h->pos, 8);
            }
            nrec++;
        }
    }
    return nrec;
}

// general_work itself over one buffer: its return value and the items it consumed
int ref_dmo_general_work(void* hv, const float* x, int n, long* consumed)
{
    Ref* h = static_cast<Ref*>(hv);
    gr_vector_int nin{ n };
    gr_vector_const_void_star in{ x };
    gr_vector_void_star o;
    const int rc = h->sink.general_work(n, nin, in, o);
    *consumed = h->sink.take_consumed();
    h->pos += n;
    h->sink.get_data();
    return rc;
}

// CDMRSlotType2::decode2087 of the 19 bits it reads (data[0], data[1], the top 3 bits of data[2]): colour code << 4 | data type
int ref_slot_type2_decode(uint32_t w19)
{
    const unsigned char b[3] = { (unsigned char)(w19 >> 11), (unsigned char)(w19 >> 3), (unsigned char)(w19 << 5) };
    CDMRSlotType2 st;
    return st.decode2087(b);
}

}  // extern "C"
