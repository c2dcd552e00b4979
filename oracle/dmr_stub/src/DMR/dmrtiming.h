// stand-in for the reference's src/DMR/dmrtiming.h (a QObject with Qt signals): records the calls gr_dmr_sink makes, so the
// shim (oracle/ref_dmr_shim.cpp) can report them.  TEST INFRASTRUCTURE ONLY (oracle/_ref build, oracle/ref_dmr.mk).
#pragma once
#include <cstdint>
#include <vector>
#include "src/DMR/constants.h"

class DMRTiming {
public:
    void set_timer(uint64_t value) { timers.push_back(value); }
    void increment_sample_counter(uint64_t n) { samples += n; increments++; }
    void set_slot_times(uint8_t sn) { slot_times.push_back(sn); }
    uint64_t samples = 0, increments = 0;
    std::vector<uint64_t> timers;
    std::vector<uint8_t> slot_times;
};
