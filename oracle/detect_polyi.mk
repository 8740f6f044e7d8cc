# oracle/detect_polyi.mk — TEST INFRASTRUCTURE ONLY (never linked into the product).
#
# Builds oracle/_ref/libnpref_polyi.so: libnpref.so's objects (the UNMODIFIED reference translation units oracle/Makefile
# compiles in place from $(REF), and ref_harness.o) plus detect_polyi_harness.cpp, which compiles src/nanopolish_detect_polyi.cpp
# in place (it #includes it) and drives its segmentation HMM, duration profile, length, QC and Bernoulli functions.  Same flags,
# one section per function, the same --gc-sections link and export list as libnpref.so: detect_polyi_main and the ReadDB / BAM
# code it reaches are dropped.
# Usage: make -C oracle -f detect_polyi.mk
include Makefile

.DEFAULT_GOAL := polyi
.PHONY: polyi

ifneq ($(wildcard $(REF)/src/nanopolish_detect_polyi.cpp),)
polyi: $(OUT)/libnpref_polyi.so
else
polyi:
	@echo "oracle: $(REF) not present (GPU box): using prebuilt $(OUT)/libnpref_polyi.so if any"
endif

$(OUT)/obj/detect_polyi_harness.o: detect_polyi_harness.cpp $(REF)/src/nanopolish_detect_polyi.cpp
	@mkdir -p $(OUT)/obj
	$(CXX) $(REFFLAGS) -ffunction-sections -fdata-sections $(REFINC) -c $< -o $@

$(OUT)/libnpref_polyi.so: $(REF_OBJS) $(REF_GC_OBJS) $(OUT)/obj/ref_harness.o $(OUT)/obj/detect_polyi_harness.o npref.map
	$(CXX) -shared -fopenmp -Wl,--gc-sections -Wl,--version-script=npref.map -o $@ $(REF_OBJS) $(REF_GC_OBJS) $(OUT)/obj/ref_harness.o $(OUT)/obj/detect_polyi_harness.o
