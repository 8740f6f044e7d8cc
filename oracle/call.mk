# oracle/call.mk — TEST INFRASTRUCTURE ONLY (never linked into the product).
#
# Builds oracle/_ref/libnpref_call.so: libnpref.so's objects (the UNMODIFIED reference translation units oracle/Makefile compiles
# in place from $(REF), and ref_harness.o), the reference's src/hmm/nanopolish_duration_model.cpp and src/thirdparty/fet.c (the
# Fisher test simple_call reaches), and call_harness.cpp, which compiles src/nanopolish_call_variants.cpp in place (it #includes it)
# so that the reference's own call_haplotype_from_candidates runs.  One symbol is wrapped (-Wl,--wrap), as in screen.mk:
# adaptive_banded_simple_event_align, through whose call in npref_abea the harness finds a read by its handle.  Same flags, one
# section per function, the same --gc-sections link and export list as libnpref.so.
# Usage: make -C oracle -f call.mk
include Makefile

.DEFAULT_GOAL := call
.PHONY: call

ifneq ($(wildcard $(REF)/src/nanopolish_call_variants.cpp),)
call: $(OUT)/libnpref_call.so
else
call:
	@echo "oracle: $(REF) not present (GPU box): using prebuilt $(OUT)/libnpref_call.so if any"
endif

CALL_WRAP := _Z34adaptive_banded_simple_event_alignR12SquiggleReadRK9PoreModelRKNSt7__cxx1112basic_stringIcSt11char_traitsIcESaIcEEE

$(OUT)/obj/call_harness.o $(OUT)/obj/call_duration_model.o: REFFLAGS += -ffunction-sections -fdata-sections
$(OUT)/obj/call_harness.o: call_harness.cpp $(REF)/src/nanopolish_call_variants.cpp
	@mkdir -p $(OUT)/obj
	$(CXX) $(REFFLAGS) $(REFINC) -c $< -o $@
$(OUT)/obj/call_duration_model.o: $(REF)/src/hmm/nanopolish_duration_model.cpp
	@mkdir -p $(OUT)/obj
	$(CXX) $(REFFLAGS) $(REFINC) -c $< -o $@
$(OUT)/obj/call_fet.o: $(REF)/src/thirdparty/fet.c
	@mkdir -p $(OUT)/obj
	$(CC) $(REFCFLAGS) -ffunction-sections -fdata-sections -I$(REF)/src/thirdparty -c $< -o $@

$(OUT)/libnpref_call.so: $(REF_OBJS) $(REF_GC_OBJS) $(OUT)/obj/ref_harness.o $(OUT)/obj/call_duration_model.o $(OUT)/obj/call_fet.o $(OUT)/obj/call_harness.o npref.map
	$(CXX) -shared -fopenmp -Wl,--gc-sections -Wl,--version-script=npref.map $(addprefix -Wl$(comma)--wrap=,$(CALL_WRAP)) -o $@ $(filter %.o,$^)
comma := ,
