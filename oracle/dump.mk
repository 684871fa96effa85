# TEST INFRASTRUCTURE -- builds the channel-dump (-go DUMP) checkers next to those of oracle/Makefile, never the product.
#
#   make -C oracle -f dump.mk refdump      -> oracle/_ref/libaisref_dump.so : ref_harness_dump.cpp + the UNMODIFIED reference objects
#   make -C oracle -f dump.mk adapterdump  -> oracle/_ref/adapter_dump_test : tests/host/adapter_dump_main.cpp (ModelGPU and the
#                                                                             reference's models with -go DUMP in one binary)
# Reuses oracle/Makefile's variables and object rules (the strict-flags reference objects under _ref/strict/).

include Makefile

.PHONY: refdump adapterdump

ifneq ($(wildcard $(S)/DSP/Model.cpp),)
refdump: $(OUT)/libaisref_dump.so
adapterdump: $(OUT)/adapter_dump_test
else
refdump adapterdump:
	@echo "reference tree $(REF) not present: using prebuilt $(OUT)/ if any"
endif

$(OUT)/strict/ref_harness_dump.o: ref_harness_dump.cpp ref_harness.cpp
	@mkdir -p $(dir $@)
	$(CXX) $(COMMON) $(STRICT) -fno-access-control -c $< -o $@

$(OUT)/libaisref_dump.so: $(OBJ_S) $(OUT)/strict/ref_harness_dump.o
	$(CXX) -shared -o $@ $^ -lpthread -ldl

$(OUT)/adapter_dump_test: ../tests/host/adapter_dump_main.cpp $(PKG)/host/ModelGPU.h ../include/aisgpu.h $(OBJ_S) $(PKG)/libaisgpu.so
	$(CXX) $(COMMON) $(STRICT) -fno-access-control -I../include -I$(PKG)/host -o $@ ../tests/host/adapter_dump_main.cpp $(OBJ_S) \
		-L$(PKG) -laisgpu -Wl,-rpath,'$$ORIGIN/../../ais-catcher_b200' -lpthread -ldl
