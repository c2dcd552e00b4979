// C-ABI shim over the reference's DMR transmit-side burst encoders, compiled UNMODIFIED from /root/reference (src/DMR/dmrframe.cpp and
// the src/MMDVM LC / FEC files behind it; oracle/ref_dmr_tx.mk, run by build()).  Each call builds one burst the way DMRControl does
// (src/DMR/dmrcontrol.cpp:80-137, 151-170) and returns DMRFrame::toByteVector.  DMRControl itself is not compiled (it needs QObject,
// Settings and Logger): the calls below set the classes up as its lines do, and restate none of the encoders.
// TEST INFRASTRUCTURE ONLY (oracle/_ref/libqrl_ref_dmr_tx.so): pins tests/dmr_tx_model.py and qrl_dmr.cu's transmit handle to the
// reference's own code (tests/test_dmr_tx_codec.py).  Nothing of the product links or loads this.
#include <cstring>
#include <vector>
#include "src/DMR/dmrframe.h"
#include "src/MMDVM/DMRLC.h"

namespace {
void copy_out(DMRFrame& f, unsigned char* out33)
{
    const std::vector<uint8_t> b = f.toByteVector();
    std::memcpy(out33, b.data(), 33);
}

CDMRLC make_lc(int flco, int fid, int options, unsigned src, unsigned dst)
{
    CDMRLC lc(FLCO(flco), src, dst);
    lc.setFID(static_cast<unsigned char>(fid));
    lc.setOptions(static_cast<unsigned char>(options));
    return lc;
}
}  // namespace

extern "C" {

// getStartCSBK's frame (dmrcontrol.cpp:99-118)
void ref_dmr_tx_csbk(int cc, int slot, unsigned src, unsigned dst, unsigned char* out33)
{
    CDMRCSBK csbk;
    csbk.setCSBKO(CSBKO_BSDWNACT);
    csbk.setCBF(0x00);
    csbk.setData1(0x00);
    csbk.setSrcId(src);
    csbk.setDstId(dst);
    DMRFrame frame(DMRFrameTypeData);
    frame.setDataType(DT_CSBK);
    frame.setColorCode(static_cast<uint8_t>(cc));
    frame.setSlotNo(static_cast<uint8_t>(slot));
    frame.constructCSBKFrame(csbk);
    copy_out(frame, out33);
}

// getVoiceHeader's (dt = DT_VOICE_LC_HEADER) or getVoiceTerminator's (DT_TERMINATOR_WITH_LC) frame for an LC (dmrcontrol.cpp:80-97, 120-128)
void ref_dmr_tx_lc(int dt, int cc, int slot, int flco, int fid, unsigned src, unsigned dst, unsigned char* out33)
{
    CDMRLC lc = make_lc(flco, fid, 0, src, dst);
    DMRFrame frame(DMRFrameTypeData);
    frame.setDataType(static_cast<uint8_t>(dt));
    frame.setColorCode(static_cast<uint8_t>(cc));
    frame.setSlotNo(static_cast<uint8_t>(slot));
    frame.constructLCFrame(&lc);
    copy_out(frame, out33);
}

// getTxAudio's voice frame (dmrcontrol.cpp:150-164): FN 0 = setVoice + addVoiceSync; FN 1-5 = setVoice + setEmbeddedData with an
// embedded-data object set from the LC (flco, fid, options, src, dst) as setLC leaves it
void ref_dmr_tx_voice(const unsigned char* audio27, int fn, int cc, int flco, int fid, int options, unsigned src, unsigned dst,
                      unsigned char* out33)
{
    unsigned char audio[27];
    std::memcpy(audio, audio27, 27);
    DMRFrame frame(DMRFrameTypeVoice);
    frame.setColorCode(static_cast<uint8_t>(cc));
    if (fn == 0) {
        frame.setFrameType(DMRFrameTypeVoiceSync);
        frame.setVoice(audio);
        frame.addVoiceSync();
    } else {
        frame.setFrameType(DMRFrameTypeVoice);
        frame.setVoice(audio);
        CDMREmbeddedData emb;
        emb.setLC(make_lc(flco, fid, options, src, dst));
        frame.setEmbeddedData(emb, static_cast<uint8_t>(fn));
    }
    copy_out(frame, out33);
}

}  // extern "C"
