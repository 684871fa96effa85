# TEST INFRASTRUCTURE -- builds the single-channel (-c X) checkers next to those of oracle/Makefile, never the product.
#
#   make -C oracle -f mode_x.mk refx      -> oracle/_ref/libaisrefx.so     : ref_harness_x.cpp + the UNMODIFIED reference objects
#   make -C oracle -f mode_x.mk adapterx  -> oracle/_ref/adapter_mode_test : tests/host/adapter_mode_main.cpp (ModelGPU in a
#                                                                            channel mode, inside the reference's block graph)
# Reuses oracle/Makefile's variables and object rules (the strict-flags reference objects under _ref/strict/).

include Makefile

.PHONY: refx adapterx

ifneq ($(wildcard $(S)/DSP/Model.cpp),)
refx: $(OUT)/libaisrefx.so
adapterx: $(OUT)/adapter_mode_test
else
refx adapterx:
	@echo "reference tree $(REF) not present: using prebuilt $(OUT)/ if any"
endif

$(OUT)/strict/ref_harness_x.o: ref_harness_x.cpp ref_harness.cpp
	@mkdir -p $(dir $@)
	$(CXX) $(COMMON) $(STRICT) -fno-access-control -c $< -o $@

$(OUT)/libaisrefx.so: $(OBJ_S) $(OUT)/strict/ref_harness_x.o
	$(CXX) -shared -o $@ $^ -lpthread -ldl

$(OUT)/adapter_mode_test: ../tests/host/adapter_mode_main.cpp $(PKG)/host/ModelGPU.h ../include/aisgpu.h $(OBJ_S) $(PKG)/libaisgpu.so
	$(CXX) $(COMMON) $(STRICT) -fno-access-control -I../include -I$(PKG)/host -o $@ ../tests/host/adapter_mode_main.cpp $(OBJ_S) \
		-L$(PKG) -laisgpu -Wl,-rpath,'$$ORIGIN/../../ais-catcher_b200' -lpthread -ldl
