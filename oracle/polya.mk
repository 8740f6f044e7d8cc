# oracle/polya.mk — TEST INFRASTRUCTURE ONLY (never linked into the product).
#
# Builds oracle/_ref/libnpref_polya.so: libnpref.so's objects (the UNMODIFIED reference translation units oracle/Makefile compiles
# in place from $(REF), and ref_harness.o) plus polya_harness.cpp, which compiles src/nanopolish_polya_estimator.cpp in place (it
# #includes it) and drives its SegmentationHMM, duration profile, length and QC functions.  Same flags, one section per function,
# the same --gc-sections link and export list as libnpref.so: polya_main and the ReadDB / BAM code it reaches are dropped.
# Usage: make -C oracle -f polya.mk
include Makefile

.DEFAULT_GOAL := polya
.PHONY: polya

ifneq ($(wildcard $(REF)/src/nanopolish_polya_estimator.cpp),)
polya: $(OUT)/libnpref_polya.so
else
polya:
	@echo "oracle: $(REF) not present (GPU box): using prebuilt $(OUT)/libnpref_polya.so if any"
endif

$(OUT)/obj/polya_harness.o: polya_harness.cpp $(REF)/src/nanopolish_polya_estimator.cpp
	@mkdir -p $(OUT)/obj
	$(CXX) $(REFFLAGS) -ffunction-sections -fdata-sections $(REFINC) -c $< -o $@

$(OUT)/libnpref_polya.so: $(REF_OBJS) $(REF_GC_OBJS) $(OUT)/obj/ref_harness.o $(OUT)/obj/polya_harness.o npref.map
	$(CXX) -shared -fopenmp -Wl,--gc-sections -Wl,--version-script=npref.map -o $@ $(REF_OBJS) $(REF_GC_OBJS) $(OUT)/obj/ref_harness.o $(OUT)/obj/polya_harness.o
