# TEST INFRASTRUCTURE -- builds the probes of the frequency-correction tests next to the checkers of oracle/Makefile, never the product.
#
#   make -C oracle -f afc.mk refafc  -> oracle/_ref/libaisref_afc.so, libaisrefx_afc.so : ref_harness_afc.cpp around ref_harness.cpp /
#                                       ref_harness_x.cpp + the UNMODIFIED reference objects (the V2 engines' state after a push)
# Reuses oracle/Makefile's variables and object rules (the strict-flags reference objects under _ref/strict/).

include Makefile

.PHONY: refafc

ifneq ($(wildcard $(S)/DSP/Model.cpp),)
refafc: $(OUT)/libaisref_afc.so $(OUT)/libaisrefx_afc.so
else
refafc:
	@echo "reference tree $(REF) not present: using prebuilt $(OUT)/ if any"
endif

$(OUT)/strict/ref_harness_afc.o: ref_harness_afc.cpp ref_harness.cpp
	@mkdir -p $(dir $@)
	$(CXX) $(COMMON) $(STRICT) -fno-access-control -c $< -o $@

$(OUT)/strict/ref_harness_afc_x.o: ref_harness_afc.cpp ref_harness_x.cpp ref_harness.cpp
	@mkdir -p $(dir $@)
	$(CXX) $(COMMON) $(STRICT) -fno-access-control -DAFC_BASE='"ref_harness_x.cpp"' -c $< -o $@

$(OUT)/libaisref_afc.so: $(OBJ_S) $(OUT)/strict/ref_harness_afc.o
	$(CXX) -shared -o $@ $^ -lpthread -ldl

$(OUT)/libaisrefx_afc.so: $(OBJ_S) $(OUT)/strict/ref_harness_afc_x.o
	$(CXX) -shared -o $@ $^ -lpthread -ldl
