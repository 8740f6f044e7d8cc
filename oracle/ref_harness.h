// oracle/ref_harness.h — TEST INFRASTRUCTURE ONLY.  What ref_harness.cpp shares with the harnesses linked beside it.
#pragma once
#include <string>

class SquiggleRead;

// the "FASTA index" ref_harness.cpp's faidx_fetch_seq double reads behind a faidx_t*: one contig held in memory
struct NprefContig { std::string name, seq; };

// the read behind a handle of npref_read_create.  C++ linkage: npref.map exports only unmangled npref_* names, so this stays
// local to each library and links only between the objects inside it
SquiggleRead* npref_read_of(int h);
