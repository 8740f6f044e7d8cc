# oracle/phase.mk — TEST INFRASTRUCTURE ONLY (never linked into the product).
#
# Builds oracle/_ref/libnpref_phase.so: libnpref.so's objects (the UNMODIFIED reference translation units oracle/Makefile compiles
# in place from $(REF), and ref_harness.o), the reference's src/common/nanopolish_bam_utils.cpp (write_bam_vardata), and
# phase_reads_harness.cpp, which compiles src/nanopolish_phase_reads.cpp in place (it #includes it) so that the reference's own
# phase_single_read runs.  One symbol is wrapped (-Wl,--wrap): the SquiggleRead constructor that loads from a ReadDB.  Same flags, one
# section per function, the same --gc-sections link and export list as libnpref.so: phase_reads_main and the ReadDB / BAM code
# it reaches are dropped.
# Usage: make -C oracle -f phase.mk
include Makefile

.DEFAULT_GOAL := phase
.PHONY: phase

ifneq ($(wildcard $(REF)/src/nanopolish_phase_reads.cpp),)
phase: $(OUT)/libnpref_phase.so
else
phase:
	@echo "oracle: $(REF) not present (GPU box): using prebuilt $(OUT)/libnpref_phase.so if any"
endif

PHASE_WRAP := _ZN12SquiggleReadC1ERKNSt7__cxx1112basic_stringIcSt11char_traitsIcESaIcEEERK6ReadDBj

$(OUT)/obj/phase_reads_harness.o $(OUT)/obj/nanopolish_bam_utils.o: REFFLAGS += -ffunction-sections -fdata-sections
$(OUT)/obj/phase_reads_harness.o: phase_reads_harness.cpp ref_harness.h $(REF)/src/nanopolish_phase_reads.cpp
	@mkdir -p $(OUT)/obj
	$(CXX) $(REFFLAGS) $(REFINC) -c $< -o $@
$(OUT)/obj/nanopolish_bam_utils.o: $(REF)/src/common/nanopolish_bam_utils.cpp
	@mkdir -p $(OUT)/obj
	$(CXX) $(REFFLAGS) $(REFINC) -c $< -o $@

$(OUT)/libnpref_phase.so: $(REF_OBJS) $(REF_GC_OBJS) $(OUT)/obj/ref_harness.o $(OUT)/obj/nanopolish_bam_utils.o $(OUT)/obj/phase_reads_harness.o npref.map
	$(CXX) -shared -fopenmp -Wl,--gc-sections -Wl,--version-script=npref.map $(addprefix -Wl$(comma)--wrap=,$(PHASE_WRAP)) -o $@ $(filter %.o,$^)
comma := ,
