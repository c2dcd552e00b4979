// C-ABI shim over the reference's M17 frame codec, compiled UNMODIFIED from /root/reference/src/M17/M17 (M17FrameDecoder,
// M17FrameEncoder, M17Transmitter, M17Golay, M17LinkSetupFrame, M17Callsign; oracle/ref_m17.mk, run by build()), plus the few lines of
// gr_modem's M17 branches that drive it (/root/reference/src/gr_modem.cpp:719-728, 1370-1440).
// TEST INFRASTRUCTURE ONLY (oracle/_ref/libqrl_ref_m17.so): pins qrl_m17.cu and qradiolink_b200/m17.py to the reference's own code
// (tests/test_m17_codec.py).  Nothing of the product links or loads this.
#include <M17/M17Callsign.hpp>
#include <M17/M17FrameDecoder.hpp>
#include <M17/M17LinkSetupFrame.hpp>
#include <M17/M17Transmitter.hpp>

#include <cstring>
#include <string>
#include <vector>

namespace {
constexpr uint32_t kStream = 0xFF5D, kLsf = 0x55F7, kEot = 0x555D555D;     // layer1framing.h:21-23

int push(const std::vector<unsigned char>& v, unsigned char* out)
{
    std::memcpy(out, v.data(), v.size());
    return static_cast<int>(v.size());
}
}  // namespace

extern "C" {

// ---------------------------------------------------------------- receive: M17FrameDecoder behind gr_modem::processReceivedData
// M17FrameDecoder's constructor leaves lsfSegmentMap uninitialised (gr_modem's `_m17_decoder()` runs that user-provided constructor,
// which zeroes nothing), so the map of the first transmission is whatever the heap held.  The shim starts from reset(), the state
// every transmission after a valid EOT starts from; the device decoder's initial state is the same.
void* ref_m17_dec_create()
{
    auto* h = new M17::M17FrameDecoder();
    h->reset();
    return h;
}
void ref_m17_dec_destroy(void* h) { delete static_cast<M17::M17FrameDecoder*>(h); }

// one deframed record {type, 46 bytes}: out56 = { uint32 type, getLsf() 30 bytes, lsf.valid(), 0, getStreamFrame() 18 bytes, 0, 0 }
// as they stand after gr_modem handled the record (an EOT record: before the reset a valid LSF triggers)
void ref_m17_dec_record(void* hv, uint32_t type, const unsigned char* payload46, unsigned char* out56)
{
    auto* h = static_cast<M17::M17FrameDecoder*>(hv);
    if (type == kStream || type == kLsf) {
        M17::frame_t frame;
        frame[0] = (type >> 8) & 0xFF;
        frame[1] = type & 0xFF;
        std::memcpy(frame.data() + 2, payload46, 46);
        h->decodeFrame(frame);
    }
    M17::M17LinkSetupFrame lsf = h->getLsf();
    M17::M17StreamFrame sf = h->getStreamFrame();
    std::memset(out56, 0, 56);
    std::memcpy(out56, &type, 4);
    std::memcpy(out56 + 4, lsf.getData(), 30);
    out56[34] = lsf.valid() ? 1 : 0;
    std::memcpy(out56 + 36, sf.getData(), 18);
    if (type == kEot && lsf.valid()) h->reset();
}

// ---------------------------------------------------------------- transmit: M17Transmitter behind gr_modem
void* ref_m17_tx_create() { return new M17::M17Transmitter(); }
void ref_m17_tx_destroy(void* h) { delete static_cast<M17::M17Transmitter*>(h); }

int ref_m17_tx_start(void* h, const char* src, const char* dst, int can, int destination_type, unsigned char* out)
{
    std::vector<unsigned char> v;
    static_cast<M17::M17Transmitter*>(h)->start(src, dst, static_cast<uint16_t>(can), destination_type, &v);
    return push(v, out);
}

// last = 0: gr_modem::transmitM17Audio; last = 1: gr_modem::endTransmission (last frame, then _tx_frame_length / 2 EOT words)
int ref_m17_tx_send(void* h, const unsigned char* payload16, int last, unsigned char* out)
{
    std::vector<unsigned char> v;
    M17::payload_t p;
    std::memcpy(p.data(), payload16, 16);
    static_cast<M17::M17Transmitter*>(h)->send(p, &v, last != 0);
    if (last)
        for (int i = 0; i < 16 / 2; i++) { v.push_back((kEot >> 8) & 0xFF); v.push_back(kEot & 0xFF); }
    return push(v, out);
}

// ---------------------------------------------------------------- LSF and callsigns
// the LSF M17Transmitter::start builds (its 30 bytes, CRC included).  start() leaves the encryption subtype and the reserved bits of
// its streamType_t uninitialised; here they are zero, as they come out of start() in this build (the stored digests pin that)
void ref_m17_lsf(const char* src, const char* dst, int can, int destination_type, unsigned char* out30)
{
    M17::M17LinkSetupFrame lsf;
    lsf.clear();
    lsf.setSource(src);
    if (destination_type == 0) {
        if (std::strlen(dst)) lsf.setDestination(std::string(dst));
    } else {
        lsf.setDestination(destination_type);
    }
    M17::streamType_t type;
    type.value = 0;
    type.fields.stream = 1;
    type.fields.dataType = 2;
    type.fields.CAN = static_cast<uint16_t>(can);
    type.fields.encType = 0;
    lsf.setType(type);
    lsf.updateCrc();
    std::memcpy(out30, lsf.getData(), 30);
}

void ref_m17_encode_callsign(const char* callsign, unsigned char* out6)
{
    M17::call_t c;
    M17::encode_callsign(callsign, c);
    std::memcpy(out6, c.data(), 6);
}

int ref_m17_decode_callsign(const unsigned char* in6, char* out, int cap)
{
    M17::call_t c;
    std::memcpy(c.data(), in6, 6);
    const std::string s = M17::decode_callsign(c);
    std::strncpy(out, s.c_str(), cap);
    return static_cast<int>(s.size());
}

}  // extern "C"
