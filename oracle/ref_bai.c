/* oracle/ref_bai.c -- TEST-ONLY checker around htslib's BAM indexer and region iterator (the copy the reference carries in
 * contrib/htslib, unmodified), built by ref_bai.mk into _ref/libnvbio_ref_bai.so:
 *   ref_bam_index    bam_index_build(path, 0): writes path + ".bai";
 *   ref_bam_query    the records a region query through path + ".bai" yields (sam_index_load, sam_itr_queryi, sam_itr_next), as
 *                    sam_format1 text. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include "htslib/sam.h"
#include "htslib/kstring.h"

int ref_bam_index(const char* path) { return bam_index_build(path, 0); }

/* the records of [beg, end) on tid that the iterator over path + ".bai" yields, as sam_format1 lines into out (at most cap bytes,
 * NUL-terminated).  Returns the number of records, -1 when the file, its header or the index cannot be read, -2 when out is too small,
 * -3 when the iterator fails. */
long long ref_bam_query(const char* path, int tid, int beg, int end, char* out, unsigned long long cap)
{
    samFile* fp = sam_open(path, "r");
    if (!fp) return -1;
    bam_hdr_t* h = sam_hdr_read(fp);
    hts_idx_t* idx = h ? sam_index_load(fp, path) : NULL;
    if (!idx) { if (h) bam_hdr_destroy(h); sam_close(fp); return -1; }
    hts_itr_t* it = sam_itr_queryi(idx, tid, beg, end);
    bam1_t* b = bam_init1();
    kstring_t s = { 0, 0, NULL };
    long long n = 0;
    unsigned long long used = 0;
    int r = -1;
    while (it && (r = sam_itr_next(fp, it, b)) >= 0) {
        s.l = 0;
        sam_format1(h, b, &s);
        if (used + s.l + 2 > cap) { n = -2; break; }
        memcpy(out + used, s.s, s.l);
        used += s.l;
        out[used++] = '\n';
        ++n;
    }
    if (n >= 0 && (!it || r < -1)) n = -3;
    if (cap) out[used < cap ? used : cap - 1] = 0;
    free(s.s);
    bam_destroy1(b);
    if (it) hts_itr_destroy(it);
    hts_idx_destroy(idx);
    bam_hdr_destroy(h);
    sam_close(fp);
    return n;
}
