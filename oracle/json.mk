# TEST INFRASTRUCTURE -- builds the full-JSON checker next to those of oracle/Makefile, never the product.
#
#   make -C oracle -f json.mk refjson -> oracle/_ref/libaisref_json.so : ref_harness_json.cpp + the UNMODIFIED reference's
#                                        JSONAIS, Serializer, Message and key tables
# Reuses oracle/Makefile's variables and object rules (the strict-flags reference objects under _ref/strict/).

include Makefile

.PHONY: refjson

ifneq ($(wildcard $(S)/DSP/Model.cpp),)
refjson: $(OUT)/libaisref_json.so
else
refjson:
	@echo "reference tree $(REF) not present: using prebuilt $(OUT)/ if any"
endif

$(OUT)/strict/ref_harness_json.o: ref_harness_json.cpp
	@mkdir -p $(dir $@)
	$(CXX) $(COMMON) $(STRICT) -fno-access-control -c $< -o $@

$(OUT)/libaisref_json.so: $(OBJ_S) $(OUT)/strict/ref_harness_json.o
	$(CXX) -shared -o $@ $^ -lpthread -ldl
