# oracle/hp.mk — TEST INFRASTRUCTURE ONLY (never linked into the product).
#
# Builds oracle/_ref/libnpref_hp.so: libnpref.so's objects (the UNMODIFIED reference translation units oracle/Makefile compiles
# in place from $(REF), and ref_harness.o), the reference's src/hmm/nanopolish_duration_model.cpp, and hp_harness.cpp, which
# compiles src/nanopolish_call_variants.cpp in place (it #includes it) so that the reference's own fix_homopolymers runs.  One
# symbol is wrapped (-Wl,--wrap): adaptive_banded_simple_event_align, through whose call in npref_abea the harness finds a read by
# its handle.  Same flags, one section per function, the same --gc-sections link and export list as libnpref.so:
# call_variants_main and the BAM / FASTA code it reaches are dropped.
# Usage: make -C oracle -f hp.mk
include Makefile

.DEFAULT_GOAL := hp
.PHONY: hp

ifneq ($(wildcard $(REF)/src/nanopolish_call_variants.cpp),)
hp: $(OUT)/libnpref_hp.so
else
hp:
	@echo "oracle: $(REF) not present (GPU box): using prebuilt $(OUT)/libnpref_hp.so if any"
endif

HP_WRAP := _Z34adaptive_banded_simple_event_alignR12SquiggleReadRK9PoreModelRKNSt7__cxx1112basic_stringIcSt11char_traitsIcESaIcEEE

$(OUT)/obj/hp_harness.o $(OUT)/obj/nanopolish_duration_model.o: REFFLAGS += -ffunction-sections -fdata-sections
$(OUT)/obj/hp_harness.o: hp_harness.cpp $(REF)/src/nanopolish_call_variants.cpp
	@mkdir -p $(OUT)/obj
	$(CXX) $(REFFLAGS) $(REFINC) -c $< -o $@
$(OUT)/obj/nanopolish_duration_model.o: $(REF)/src/hmm/nanopolish_duration_model.cpp
	@mkdir -p $(OUT)/obj
	$(CXX) $(REFFLAGS) $(REFINC) -c $< -o $@

$(OUT)/libnpref_hp.so: $(REF_OBJS) $(REF_GC_OBJS) $(OUT)/obj/ref_harness.o $(OUT)/obj/nanopolish_duration_model.o $(OUT)/obj/hp_harness.o npref.map
	$(CXX) -shared -fopenmp -Wl,--gc-sections -Wl,--version-script=npref.map $(addprefix -Wl$(comma)--wrap=,$(HP_WRAP)) -o $@ $(filter %.o,$^)
comma := ,
