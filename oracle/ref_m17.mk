# Builds oracle/_ref/libqrl_ref_m17.so where the reference tree is present: the M17 frame codec of the reference's src/M17/M17,
# compiled UNMODIFIED where it lies, behind ref_m17_shim.cpp (gr_modem's M17 branches).  Test infrastructure only
# (tests/test_m17_codec.py); nothing is copied into the repository.  Run by __graft_entry__.build(): make -C oracle -f ref_m17.mk
REF ?= /root/reference
REF_M17 = M17FrameDecoder.cpp M17FrameEncoder.cpp M17Transmitter.cpp M17Golay.cpp M17LinkSetupFrame.cpp M17Callsign.cpp

all:
	@if [ -f $(REF)/src/M17/M17/M17FrameDecoder.cpp ]; then mkdir -p _ref && \
	g++ -O2 -std=gnu++17 -fPIC -shared -w -I$(REF)/src/M17 -o _ref/libqrl_ref_m17.so ref_m17_shim.cpp $(addprefix $(REF)/src/M17/M17/,$(REF_M17)) && \
	echo "built _ref/libqrl_ref_m17.so"; else echo "reference tree absent: using prebuilt oracle/_ref/libqrl_ref_m17.so if any"; fi

.PHONY: all
