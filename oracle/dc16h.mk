# TEST INFRASTRUCTURE -- builds the DC16H (12 bytes per sample) checkers next to those of oracle/Makefile, never the product.
#
#   make -C oracle -f dc16h.mk refdc16h      -> oracle/_ref/libaisref_dc16h.so, libaisrefx_dc16h.so, libaisrefd_dc16h.so :
#                                               ref_harness_dc16h.cpp around ref_harness.cpp / ref_harness_x.cpp /
#                                               ref_harness_disc.cpp + the UNMODIFIED reference objects
#   make -C oracle -f dc16h.mk adapterdc16h  -> oracle/_ref/adapter_dc16h_test : tests/host/adapter_dc16h_main.cpp (ModelGPU and the
#                                               reference's models on Format::DC16H buffers in one binary)
# Reuses oracle/Makefile's variables and object rules (the strict-flags reference objects under _ref/strict/).

include Makefile

.PHONY: refdc16h adapterdc16h

ifneq ($(wildcard $(S)/DSP/Model.cpp),)
refdc16h: $(OUT)/libaisref_dc16h.so $(OUT)/libaisrefx_dc16h.so $(OUT)/libaisrefd_dc16h.so
adapterdc16h: $(OUT)/adapter_dc16h_test
else
refdc16h adapterdc16h:
	@echo "reference tree $(REF) not present: using prebuilt $(OUT)/ if any"
endif

$(OUT)/strict/ref_harness_dc16h.o: ref_harness_dc16h.cpp ref_harness.cpp
	@mkdir -p $(dir $@)
	$(CXX) $(COMMON) $(STRICT) -fno-access-control -c $< -o $@

$(OUT)/strict/ref_harness_dc16h_x.o: ref_harness_dc16h.cpp ref_harness_x.cpp ref_harness.cpp
	@mkdir -p $(dir $@)
	$(CXX) $(COMMON) $(STRICT) -fno-access-control -DDC16H_BASE='"ref_harness_x.cpp"' -c $< -o $@

$(OUT)/strict/ref_harness_dc16h_disc.o: ref_harness_dc16h.cpp ref_harness_disc.cpp ref_harness.cpp
	@mkdir -p $(dir $@)
	$(CXX) $(COMMON) $(STRICT) -fno-access-control -DDC16H_BASE='"ref_harness_disc.cpp"' -c $< -o $@

$(OUT)/libaisref_dc16h.so: $(OBJ_S) $(OUT)/strict/ref_harness_dc16h.o
	$(CXX) -shared -o $@ $^ -lpthread -ldl

$(OUT)/libaisrefx_dc16h.so: $(OBJ_S) $(OUT)/strict/ref_harness_dc16h_x.o
	$(CXX) -shared -o $@ $^ -lpthread -ldl

$(OUT)/libaisrefd_dc16h.so: $(OBJ_S) $(OUT)/strict/ref_harness_dc16h_disc.o
	$(CXX) -shared -o $@ $^ -lpthread -ldl

$(OUT)/adapter_dc16h_test: ../tests/host/adapter_dc16h_main.cpp $(PKG)/host/ModelGPU.h ../include/aisgpu.h $(OBJ_S) $(PKG)/libaisgpu.so
	$(CXX) $(COMMON) $(STRICT) -fno-access-control -I../include -I$(PKG)/host -o $@ ../tests/host/adapter_dc16h_main.cpp $(OBJ_S) \
		-L$(PKG) -laisgpu -Wl,-rpath,'$$ORIGIN/../../ais-catcher_b200' -lpthread -ldl
