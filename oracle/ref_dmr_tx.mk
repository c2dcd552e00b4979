# Builds oracle/_ref/libqrl_ref_dmr_tx.so where the reference tree is present: DMRFrame and the src/MMDVM LC and FEC code its transmit
# side uses (CDMRFullLC, CDMRCSBK, CDMREmbeddedData, CDMREMB, CDMRLC, CDMRSlotType, CSync), compiled UNMODIFIED where they lie, behind
# ref_dmr_tx_shim.cpp.  Test infrastructure only (tests/test_dmr_tx_codec.py); nothing is copied into the repository.  _FORTIFY_SOURCE
# is off for the reason ref_dmr.mk gives (Log.cpp).  Run by __graft_entry__.build(): make -C oracle -f ref_dmr_tx.mk
REF ?= /root/reference
REF_DMR_TX = src/DMR/dmrframe.cpp \
             $(addprefix src/MMDVM/,AMBEFEC.cpp BPTC19696.cpp CRC.cpp DMRCSBK.cpp DMRDataHeader.cpp DMREMB.cpp DMREmbeddedData.cpp DMRFullLC.cpp \
             DMRLC.cpp DMRSlotType.cpp DMRTrellis.cpp Golay2087.cpp Golay24128.cpp Hamming.cpp QR1676.cpp RS129.cpp Sync.cpp Utils.cpp Log.cpp \
             DMRData.cpp)

all:
	@if [ -f $(REF)/src/DMR/dmrframe.cpp ]; then mkdir -p _ref && \
	g++ -O2 -U_FORTIFY_SOURCE -D_FORTIFY_SOURCE=0 -std=gnu++17 -fPIC -shared -w -Idmr_stub -Igr_stub -I$(REF) -I$(REF)/src/MMDVM -o _ref/libqrl_ref_dmr_tx.so ref_dmr_tx_shim.cpp \
	    $(addprefix $(REF)/,$(REF_DMR_TX)) && echo "built _ref/libqrl_ref_dmr_tx.so"; \
	else echo "reference tree absent: using prebuilt oracle/_ref/libqrl_ref_dmr_tx.so if any"; fi

.PHONY: all
