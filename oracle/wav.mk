# TEST INFRASTRUCTURE -- builds the WAV-input checker next to those of oracle/Makefile, never the product.
#
#   make -C oracle -f wav.mk refwav  -> oracle/_ref/libaisref_wav.so : ref_harness_wav.cpp + the UNMODIFIED reference's
#                                       Device/FileWAV.cpp and objects
# Reuses oracle/Makefile's variables and object rules (the strict-flags reference objects under _ref/strict/).

include Makefile

.PHONY: refwav

ifneq ($(wildcard $(S)/DSP/Model.cpp),)
refwav: $(OUT)/libaisref_wav.so
else
refwav:
	@echo "reference tree $(REF) not present: using prebuilt $(OUT)/ if any"
endif

$(OUT)/strict/ref_harness_wav.o: ref_harness_wav.cpp
	@mkdir -p $(dir $@)
	$(CXX) $(COMMON) $(STRICT) -fno-access-control -c $< -o $@

$(OUT)/libaisref_wav.so: $(OBJ_S) $(OUT)/strict/Device/FileWAV.o $(OUT)/strict/ref_harness_wav.o
	$(CXX) -shared -o $@ $^ -lpthread -ldl
