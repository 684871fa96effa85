# TEST INFRASTRUCTURE -- builds the FM-discriminator input model (-m 3) checkers next to those of oracle/Makefile, never the product.
#
#   make -C oracle -f disc.mk refd      -> oracle/_ref/libaisrefd.so      : ref_harness_disc.cpp + the UNMODIFIED reference objects
#   make -C oracle -f disc.mk adapterd  -> oracle/_ref/adapter_disc_test  : tests/host/adapter_disc_main.cpp (ModelGPU(-m 3) and the
#                                                                           reference's ModelDiscriminator in the same block graph)
# Reuses oracle/Makefile's variables and object rules (the strict-flags reference objects under _ref/strict/).

include Makefile

.PHONY: refd adapterd

ifneq ($(wildcard $(S)/DSP/Model.cpp),)
refd: $(OUT)/libaisrefd.so
adapterd: $(OUT)/adapter_disc_test
else
refd adapterd:
	@echo "reference tree $(REF) not present: using prebuilt $(OUT)/ if any"
endif

$(OUT)/strict/ref_harness_disc.o: ref_harness_disc.cpp ref_harness.cpp
	@mkdir -p $(dir $@)
	$(CXX) $(COMMON) $(STRICT) -fno-access-control -c $< -o $@

$(OUT)/libaisrefd.so: $(OBJ_S) $(OUT)/strict/ref_harness_disc.o
	$(CXX) -shared -o $@ $^ -lpthread -ldl

$(OUT)/adapter_disc_test: ../tests/host/adapter_disc_main.cpp $(PKG)/host/ModelGPU.h ../include/aisgpu.h $(OBJ_S) $(PKG)/libaisgpu.so
	$(CXX) $(COMMON) $(STRICT) -fno-access-control -I../include -I$(PKG)/host -o $@ ../tests/host/adapter_disc_main.cpp $(OBJ_S) \
		-L$(PKG) -laisgpu -Wl,-rpath,'$$ORIGIN/../../ais-catcher_b200' -lpthread -ldl
