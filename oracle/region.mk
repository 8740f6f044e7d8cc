# oracle/region.mk — TEST INFRASTRUCTURE ONLY (never linked into the product).
#
# Builds oracle/_ref/libnpref_region.so: every object of libnpref_call.so (call.mk: the reference translation units compiled in place,
# ref_harness.o, the duration model, fet.c, and call_harness.o, the one in-place copy of src/nanopolish_call_variants.cpp) plus
# region_harness.cpp, which runs the reference's own get_variants_in_region and read_variants_for_region and the default mode of a
# region call through call_harness.cpp's npref_call_haplotype.  The same wrapped symbol, flags, section GC and export list.
# Usage: make -C oracle -f region.mk
include call.mk

.DEFAULT_GOAL := region
.PHONY: region

ifneq ($(wildcard $(REF)/src/nanopolish_call_variants.cpp),)
region: $(OUT)/libnpref_region.so
else
region:
	@echo "oracle: $(REF) not present (GPU box): using prebuilt $(OUT)/libnpref_region.so if any"
endif

$(OUT)/obj/region_harness.o: REFFLAGS += -ffunction-sections -fdata-sections
$(OUT)/obj/region_harness.o: region_harness.cpp
	@mkdir -p $(OUT)/obj
	$(CXX) $(REFFLAGS) $(REFINC) -c $< -o $@

$(OUT)/libnpref_region.so: $(REF_OBJS) $(REF_GC_OBJS) $(OUT)/obj/ref_harness.o $(OUT)/obj/call_duration_model.o $(OUT)/obj/call_fet.o $(OUT)/obj/call_harness.o $(OUT)/obj/region_harness.o npref.map
	$(CXX) -shared -fopenmp -Wl,--gc-sections -Wl,--version-script=npref.map $(addprefix -Wl$(comma)--wrap=,$(CALL_WRAP)) -o $@ $(filter %.o,$^)
