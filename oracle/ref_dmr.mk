# Builds oracle/_ref/libqrl_ref_dmr.so where the reference tree is present: gr_dmr_sink, DMRFrame and the src/MMDVM FEC and LC code
# they use, compiled UNMODIFIED where they lie, behind ref_dmr_shim.cpp.  dmr_stub/ (a DMRTiming that records its calls, and the pmt
# calls of rx_time tags) comes ahead of gr_stub/ on the include path.  Test infrastructure only (tests/test_dmr_codec.py); nothing is
# copied into the repository.  _FORTIFY_SOURCE is off: Log.cpp passes vsnprintf a size of 500 for what is left of a 501-byte buffer, which
# the fortified libc aborts on although no message comes near that length.  Run by __graft_entry__.build(): make -C oracle -f ref_dmr.mk
REF ?= /root/reference
REF_DMR = src/gr/gr_dmr_sink.cpp src/DMR/dmrframe.cpp \
          $(addprefix src/MMDVM/,AMBEFEC.cpp BPTC19696.cpp CRC.cpp DMRCSBK.cpp DMRDataHeader.cpp DMREMB.cpp DMREmbeddedData.cpp DMRFullLC.cpp \
          DMRLC.cpp DMRSlotType.cpp DMRTrellis.cpp Golay2087.cpp Golay24128.cpp Hamming.cpp QR1676.cpp RS129.cpp Sync.cpp Utils.cpp Log.cpp \
          DMRData.cpp)

all:
	@if [ -f $(REF)/src/gr/gr_dmr_sink.cpp ]; then mkdir -p _ref && \
	g++ -O2 -U_FORTIFY_SOURCE -D_FORTIFY_SOURCE=0 -std=gnu++17 -fPIC -shared -w -Idmr_stub -Igr_stub -I$(REF) -I$(REF)/src/MMDVM -o _ref/libqrl_ref_dmr.so ref_dmr_shim.cpp \
	    $(addprefix $(REF)/,$(REF_DMR)) && echo "built _ref/libqrl_ref_dmr.so"; \
	else echo "reference tree absent: using prebuilt oracle/_ref/libqrl_ref_dmr.so if any"; fi

.PHONY: all
