# oracle/polya.mk — TEST INFRASTRUCTURE ONLY (never linked into the product).
#
# Builds the reference's two poly(A) tail callers, each as libnpref.so's objects (the UNMODIFIED reference translation units
# oracle/Makefile compiles in place from $(REF), and ref_harness.o) plus one harness:
#   oracle/_ref/libnpref_polya.so  polya_harness.cpp, which compiles src/nanopolish_polya_estimator.cpp in place (it #includes
#                                  it) and drives its SegmentationHMM, duration profile, length and QC functions
#   oracle/_ref/libnpref_polyi.so  detect_polyi_harness.cpp, which compiles src/nanopolish_detect_polyi.cpp in place and drives
#                                  its segmentation HMM, duration profile, length, QC and Bernoulli functions
# The two reference units both define the option parsers and usage strings of their commands, so each has its own harness and
# library.  Same flags, one section per function, the same --gc-sections link and export list as libnpref.so: polya_main,
# detect_polyi_main and the ReadDB / BAM code they reach are dropped.
# Usage: make -C oracle -f polya.mk
include Makefile

.DEFAULT_GOAL := tails
.PHONY: tails polya polyi
tails: polya polyi

ifneq ($(wildcard $(REF)/src/nanopolish_polya_estimator.cpp),)
polya: $(OUT)/libnpref_polya.so
else
polya:
	@echo "oracle: $(REF) not present (GPU box): using prebuilt $(OUT)/libnpref_polya.so if any"
endif

ifneq ($(wildcard $(REF)/src/nanopolish_detect_polyi.cpp),)
polyi: $(OUT)/libnpref_polyi.so
else
polyi:
	@echo "oracle: $(REF) not present (GPU box): using prebuilt $(OUT)/libnpref_polyi.so if any"
endif

TAIL_HARNESSES := $(OUT)/obj/polya_harness.o $(OUT)/obj/detect_polyi_harness.o
$(TAIL_HARNESSES): REFFLAGS += -ffunction-sections -fdata-sections
$(OUT)/obj/polya_harness.o: $(REF)/src/nanopolish_polya_estimator.cpp
$(OUT)/obj/detect_polyi_harness.o: $(REF)/src/nanopolish_detect_polyi.cpp

$(OUT)/libnpref_polya.so: $(OUT)/obj/polya_harness.o
$(OUT)/libnpref_polyi.so: $(OUT)/obj/detect_polyi_harness.o
$(OUT)/libnpref_polya.so $(OUT)/libnpref_polyi.so: $(REF_OBJS) $(REF_GC_OBJS) $(OUT)/obj/ref_harness.o npref.map
	$(CXX) -shared -fopenmp -Wl,--gc-sections -Wl,--version-script=npref.map -o $@ $(filter %.o,$^)
