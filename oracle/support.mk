# oracle/support.mk — TEST INFRASTRUCTURE ONLY (never linked into the product).
#
# Builds oracle/_ref/libnpref_support.so: libnpref.so's objects (the UNMODIFIED reference translation units oracle/Makefile compiles
# in place from $(REF), among them src/common/nanopolish_variant.cpp with annotate_variants_with_all_support, and ref_harness.o)
# and support_harness.cpp, which runs that function on a hand-built AlignmentDB.  One symbol is wrapped (-Wl,--wrap):
# adaptive_banded_simple_event_align, through whose call in npref_abea the harness finds a read by its handle.  Same flags, one
# section per function, the same --gc-sections link and export list as libnpref.so.
# Usage: make -C oracle -f support.mk
include Makefile

.DEFAULT_GOAL := support
.PHONY: support

ifneq ($(wildcard $(REF)/src/common/nanopolish_variant.cpp),)
support: $(OUT)/libnpref_support.so
else
support:
	@echo "oracle: $(REF) not present (GPU box): using prebuilt $(OUT)/libnpref_support.so if any"
endif

SUPPORT_WRAP := _Z34adaptive_banded_simple_event_alignR12SquiggleReadRK9PoreModelRKNSt7__cxx1112basic_stringIcSt11char_traitsIcESaIcEEE

$(OUT)/obj/support_harness.o: REFFLAGS += -ffunction-sections -fdata-sections
$(OUT)/obj/support_harness.o: support_harness.cpp $(REF)/src/common/nanopolish_variant.cpp
	@mkdir -p $(OUT)/obj
	$(CXX) $(REFFLAGS) $(REFINC) -c $< -o $@

$(OUT)/libnpref_support.so: $(REF_OBJS) $(REF_GC_OBJS) $(OUT)/obj/ref_harness.o $(OUT)/obj/support_harness.o npref.map
	$(CXX) -shared -fopenmp -Wl,--gc-sections -Wl,--version-script=npref.map $(addprefix -Wl$(comma)--wrap=,$(SUPPORT_WRAP)) -o $@ $(filter %.o,$^)
comma := ,
