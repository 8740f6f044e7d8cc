# oracle/ref_types.mk — TEST INFRASTRUCTURE ONLY (never linked into the product).
#
# Builds oracle/_ref/libnpref_types.so: libnpref.so's objects (the UNMODIFIED reference translation units oracle/Makefile compiles in
# place from $(REF), and ref_harness.o) plus ref_types_harness.cpp, which runs score_variant_thresholded with any list of methylation
# types.  Same flags, same --gc-sections link and export list as libnpref.so.  Usage: make -C oracle -f ref_types.mk
include Makefile

.DEFAULT_GOAL := types
.PHONY: types

ifneq ($(wildcard $(REF)/src/hmm/nanopolish_profile_hmm.cpp),)
types: $(OUT)/libnpref_types.so
else
types:
	@echo "oracle: $(REF) not present (GPU box): using prebuilt $(OUT)/libnpref_types.so if any"
endif

$(OUT)/obj/ref_types_harness.o: ref_types_harness.cpp
	@mkdir -p $(OUT)/obj
	$(CXX) $(REFFLAGS) $(REFINC) -c $< -o $@

$(OUT)/libnpref_types.so: $(REF_OBJS) $(REF_GC_OBJS) $(OUT)/obj/ref_harness.o $(OUT)/obj/ref_types_harness.o npref.map
	$(CXX) -shared -fopenmp -Wl,--gc-sections -Wl,--version-script=npref.map -o $@ $(REF_OBJS) $(REF_GC_OBJS) $(OUT)/obj/ref_harness.o $(OUT)/obj/ref_types_harness.o
