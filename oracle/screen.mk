# oracle/screen.mk — TEST INFRASTRUCTURE ONLY (never linked into the product).
#
# Builds oracle/_ref/libnpref_screen.so: libnpref.so's objects (the UNMODIFIED reference translation units oracle/Makefile compiles
# in place from $(REF), and ref_harness.o), the reference's src/hmm/nanopolish_duration_model.cpp, and screen_harness.cpp, which
# compiles src/nanopolish_call_variants.cpp in place (it #includes it) so that the reference's own
# screen_variants_by_score and expand_variants run (the duration model is linked because the same TU's fix_homopolymers names it).  One
# symbol is wrapped (-Wl,--wrap): adaptive_banded_simple_event_align, through whose call in npref_abea the harness finds a read by
# its handle.  Same flags, one section per function, the same --gc-sections link and export list as libnpref.so:
# call_variants_main and the BAM / FASTA code it reaches are dropped.
# Usage: make -C oracle -f screen.mk
include Makefile

.DEFAULT_GOAL := screen
.PHONY: screen

ifneq ($(wildcard $(REF)/src/nanopolish_call_variants.cpp),)
screen: $(OUT)/libnpref_screen.so
else
screen:
	@echo "oracle: $(REF) not present (GPU box): using prebuilt $(OUT)/libnpref_screen.so if any"
endif

SCREEN_WRAP := _Z34adaptive_banded_simple_event_alignR12SquiggleReadRK9PoreModelRKNSt7__cxx1112basic_stringIcSt11char_traitsIcESaIcEEE

$(OUT)/obj/screen_harness.o $(OUT)/obj/nanopolish_duration_model.o: REFFLAGS += -ffunction-sections -fdata-sections
$(OUT)/obj/screen_harness.o: screen_harness.cpp $(REF)/src/nanopolish_call_variants.cpp
	@mkdir -p $(OUT)/obj
	$(CXX) $(REFFLAGS) $(REFINC) -c $< -o $@
$(OUT)/obj/nanopolish_duration_model.o: $(REF)/src/hmm/nanopolish_duration_model.cpp
	@mkdir -p $(OUT)/obj
	$(CXX) $(REFFLAGS) $(REFINC) -c $< -o $@

$(OUT)/libnpref_screen.so: $(REF_OBJS) $(REF_GC_OBJS) $(OUT)/obj/ref_harness.o $(OUT)/obj/nanopolish_duration_model.o $(OUT)/obj/screen_harness.o npref.map
	$(CXX) -shared -fopenmp -Wl,--gc-sections -Wl,--version-script=npref.map $(addprefix -Wl$(comma)--wrap=,$(SCREEN_WRAP)) -o $@ $(filter %.o,$^)
comma := ,
