// oracle/ref_bns.cpp -- TEST-ONLY: nvbio's own save_bns (nvbio/basic/bnt.cpp:37-80), the writer of BWA's .ann / .amb files, behind a
// C entry point, built by ref_bam.mk into _ref/libnvbio_ref_bns.so.
#include <nvbio/basic/bnt.h>
#include <string.h>

// n_seqs sequences: names / annotations are '\n'-separated lists; offsets, lengths and gis one per sequence.  Writes <prefix>.ann and
// <prefix>.amb (no ambiguities).  Returns 0, or -1 when a file cannot be written.
extern "C" int ref_save_bns(const char* prefix, int n_seqs, const char* names, const char* annos, const long long* offsets,
                            const int* lengths, const unsigned* gis, long long l_pac, unsigned seed)
{
    nvbio::BNTSeq bns;
    bns.l_pac = l_pac; bns.n_seqs = n_seqs; bns.seed = seed; bns.n_holes = 0;
    bns.anns_data.resize(n_seqs);
    bns.anns_info.resize(n_seqs);
    const char* p = names;
    const char* q = annos;
    for (int i = 0; i < n_seqs; ++i) {
        const char* e = strchr(p, '\n');
        bns.anns_info[i].name.assign(p, e ? (size_t)(e - p) : strlen(p));
        p = e ? e + 1 : p + strlen(p);
        const char* f = strchr(q, '\n');
        bns.anns_info[i].anno.assign(q, f ? (size_t)(f - q) : strlen(q));
        q = f ? f + 1 : q + strlen(q);
        bns.anns_data[i].offset = offsets[i]; bns.anns_data[i].len = lengths[i]; bns.anns_data[i].n_ambs = 0; bns.anns_data[i].gi = gis[i];
    }
    try { nvbio::save_bns(bns, prefix); } catch (...) { return -1; }
    return 0;
}
