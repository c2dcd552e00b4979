# Builds oracle/_ref/libqrl_ref_dmr_dmo.so where the reference tree is present: gr_dmr_dmo_sink, CDMRSlotType2, DMRFrame and the
# src/MMDVM FEC and LC code ref_dmr.mk lists, compiled UNMODIFIED where they lie, behind ref_dmr_dmo_shim.cpp.  gr_dmr_dmo_sink.cpp
# returns gr::block::WORK_CALLED_PRODUCE, which the shared runtime stand-in (gr_stub/) does not declare: this build defines it on the
# command line with GNU Radio's value, -2 (general_work's "I called produce() myself").  Test infrastructure only
# (tests/test_dmr_dmo_codec.py); nothing is copied into the repository.  _FORTIFY_SOURCE is off for the reason ref_dmr.mk gives
# (Log.cpp).  Run by __graft_entry__.build(): make -C oracle -f ref_dmr_dmo.mk
REF ?= /root/reference
REF_DMR_DMO = src/gr/gr_dmr_dmo_sink.cpp src/DMR/dmrframe.cpp \
              $(addprefix src/MMDVM/,AMBEFEC.cpp BPTC19696.cpp CRC.cpp DMRCSBK.cpp DMRDataHeader.cpp DMREMB.cpp DMREmbeddedData.cpp \
              DMRFullLC.cpp DMRLC.cpp DMRSlotType.cpp DMRSlotType2.cpp DMRTrellis.cpp Golay2087.cpp Golay24128.cpp Hamming.cpp QR1676.cpp \
              RS129.cpp Sync.cpp Utils.cpp Log.cpp DMRData.cpp)

all:
	@if [ -f $(REF)/src/gr/gr_dmr_dmo_sink.cpp ]; then mkdir -p _ref && \
	g++ -O2 -U_FORTIFY_SOURCE -D_FORTIFY_SOURCE=0 -std=gnu++17 -fPIC -shared -w -DWORK_CALLED_PRODUCE=-2 -Idmr_stub -Igr_stub -I$(REF) -I$(REF)/src/MMDVM -o _ref/libqrl_ref_dmr_dmo.so ref_dmr_dmo_shim.cpp \
	    $(addprefix $(REF)/,$(REF_DMR_DMO)) && echo "built _ref/libqrl_ref_dmr_dmo.so"; \
	else echo "reference tree absent: using prebuilt oracle/_ref/libqrl_ref_dmr_dmo.so if any"; fi

.PHONY: all
