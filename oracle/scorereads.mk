# oracle/scorereads.mk — TEST INFRASTRUCTURE ONLY (never linked into the product).
#
# Builds oracle/_ref/libnpref_scorereads.so: libnpref.so's objects (the UNMODIFIED reference translation units oracle/Makefile
# compiles in place from $(REF), and ref_harness.o) and scorereads_harness.cpp, which compiles src/nanopolish_scorereads.cpp in
# place (it #includes it) so that the reference's own model_score runs, with TransitionParameters' training (already among
# libnpref.so's objects).  Same flags, one section per function, the same --gc-sections link and export list as
# libnpref.so: scorereads_main and the htslib / ReadDB code it reaches are dropped.
# Usage: make -C oracle -f scorereads.mk
include Makefile

.DEFAULT_GOAL := scorereads
.PHONY: scorereads

ifneq ($(wildcard $(REF)/src/nanopolish_scorereads.cpp),)
scorereads: $(OUT)/libnpref_scorereads.so
else
scorereads:
	@echo "oracle: $(REF) not present (GPU box): using prebuilt $(OUT)/libnpref_scorereads.so if any"
endif

$(OUT)/obj/scorereads_harness.o: REFFLAGS += -ffunction-sections -fdata-sections
$(OUT)/obj/scorereads_harness.o: scorereads_harness.cpp ref_harness.h $(REF)/src/nanopolish_scorereads.cpp
	@mkdir -p $(OUT)/obj
	$(CXX) $(REFFLAGS) $(REFINC) -c $< -o $@

$(OUT)/libnpref_scorereads.so: $(REF_OBJS) $(REF_GC_OBJS) $(OUT)/obj/ref_harness.o $(OUT)/obj/scorereads_harness.o npref.map
	$(CXX) -shared -fopenmp -Wl,--gc-sections -Wl,--version-script=npref.map -o $@ $(filter %.o,$^)
