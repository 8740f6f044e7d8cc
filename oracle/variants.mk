# oracle/variants.mk — TEST INFRASTRUCTURE ONLY (never linked into the product).
#
# Builds oracle/_ref/libnpref_variants.so: libnpref.so's objects (the UNMODIFIED reference translation units oracle/Makefile compiles
# in place from $(REF), among them src/common/nanopolish_variant.cpp and src/alignment/nanopolish_alignment_db.cpp, and ref_harness.o),
# the reference's src/hmm/nanopolish_duration_model.cpp and src/thirdparty/fet.c (the Fisher test simple_call reaches), and
# variants_harness.cpp, which compiles src/nanopolish_call_variants.cpp in place (it #includes it) so that the reference's own
# fix_homopolymers, screen_variants_by_score, expand_variants and call_haplotype_from_candidates run.  Same flags, one section per
# function, the same --gc-sections link and export list as libnpref.so: call_variants_main and the BAM / FASTA code it reaches are
# dropped.
# Usage: make -C oracle -f variants.mk
include Makefile

.DEFAULT_GOAL := variants
.PHONY: variants

ifneq ($(wildcard $(REF)/src/nanopolish_call_variants.cpp),)
variants: $(OUT)/libnpref_variants.so
else
variants:
	@echo "oracle: $(REF) not present (GPU box): using prebuilt $(OUT)/libnpref_variants.so if any"
endif

VARIANTS_OBJS := $(OUT)/obj/nanopolish_duration_model.o $(OUT)/obj/fet.o $(OUT)/obj/variants_harness.o
$(VARIANTS_OBJS): REFFLAGS += -ffunction-sections -fdata-sections
$(OUT)/obj/variants_harness.o: variants_harness.cpp ref_harness.h $(REF)/src/nanopolish_call_variants.cpp
	@mkdir -p $(OUT)/obj
	$(CXX) $(REFFLAGS) $(REFINC) -c $< -o $@
$(OUT)/obj/nanopolish_duration_model.o: $(REF)/src/hmm/nanopolish_duration_model.cpp
	@mkdir -p $(OUT)/obj
	$(CXX) $(REFFLAGS) $(REFINC) -c $< -o $@
$(OUT)/obj/fet.o: $(REF)/src/thirdparty/fet.c
	@mkdir -p $(OUT)/obj
	$(CC) $(REFCFLAGS) -ffunction-sections -fdata-sections -I$(REF)/src/thirdparty -c $< -o $@

$(OUT)/libnpref_variants.so: $(REF_OBJS) $(REF_GC_OBJS) $(OUT)/obj/ref_harness.o $(VARIANTS_OBJS) npref.map
	$(CXX) -shared -fopenmp -Wl,--gc-sections -Wl,--version-script=npref.map -o $@ $(filter %.o,$^)
