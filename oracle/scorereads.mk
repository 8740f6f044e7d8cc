# oracle/scorereads.mk — TEST INFRASTRUCTURE ONLY (never linked into the product).
#
# Builds oracle/_ref/libnpref_scorereads.so: libnpref.so's objects (the UNMODIFIED reference translation units oracle/Makefile
# compiles in place from $(REF), and ref_harness.o) and scorereads_harness.cpp, which compiles src/nanopolish_scorereads.cpp in
# place (it #includes it) so that the reference's own model_score runs, with TransitionParameters' training (already among
# libnpref.so's objects).  One symbol is wrapped (-Wl,--wrap): adaptive_banded_simple_event_align, through whose call in npref_abea
# the harness finds a read by its handle.  Same flags, one section per function, the same --gc-sections link and export list as
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

SR_WRAP := _Z34adaptive_banded_simple_event_alignR12SquiggleReadRK9PoreModelRKNSt7__cxx1112basic_stringIcSt11char_traitsIcESaIcEEE

$(OUT)/obj/scorereads_harness.o: REFFLAGS += -ffunction-sections -fdata-sections
$(OUT)/obj/scorereads_harness.o: scorereads_harness.cpp $(REF)/src/nanopolish_scorereads.cpp
	@mkdir -p $(OUT)/obj
	$(CXX) $(REFFLAGS) $(REFINC) -c $< -o $@

$(OUT)/libnpref_scorereads.so: $(REF_OBJS) $(REF_GC_OBJS) $(OUT)/obj/ref_harness.o $(OUT)/obj/scorereads_harness.o npref.map
	$(CXX) -shared -fopenmp -Wl,--gc-sections -Wl,--version-script=npref.map $(addprefix -Wl$(comma)--wrap=,$(SR_WRAP)) -o $@ $(filter %.o,$^)
comma := ,
