# TEST INFRASTRUCTURE -- builds the output-record checker next to those of oracle/Makefile, never the product.
#
#   make -C oracle -f fmt.mk reffmt -> oracle/_ref/libaisref_fmt.so : ref_harness_fmt.cpp + the UNMODIFIED reference's
#                                      OutputMessage::formatInto, Message, JSONAIS, Serializer and key tables
# Reuses oracle/Makefile's variables and object rules (the strict-flags reference objects under _ref/strict/).

include Makefile

.PHONY: reffmt

ifneq ($(wildcard $(S)/DSP/Model.cpp),)
reffmt: $(OUT)/libaisref_fmt.so
else
reffmt:
	@echo "reference tree $(REF) not present: using prebuilt $(OUT)/ if any"
endif

$(OUT)/strict/ref_harness_fmt.o: ref_harness_fmt.cpp
	@mkdir -p $(dir $@)
	$(CXX) $(COMMON) $(STRICT) -fno-access-control -c $< -o $@

$(OUT)/libaisref_fmt.so: $(OBJ_S) $(OUT)/strict/ref_harness_fmt.o
	$(CXX) -shared -Wl,--no-undefined -o $@ $^ -lpthread -ldl
