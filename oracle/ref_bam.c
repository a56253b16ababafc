/* oracle/ref_bam.c -- TEST-ONLY checker around htslib (the copy the reference carries in contrib/htslib), built by ref_bam.mk into
 * _ref/libnvbio_ref_bam.so.  htslib is the authority on the BAM record layout, the bin and the typing of integer tags:
 *   ref_bam_encode   SAM header text + SAM lines -> the bytes bam_write1 writes for each line (sam_parse1, then an uncompressed BGZF
 *                    stream, "wu", read back);
 *   ref_bam_format   a .bam file -> the SAM text sam_format1 gives for each record (one line each);
 *   ref_reg2bin      hts_reg2bin(beg, end, 14, 5). */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include "htslib/sam.h"
#include "htslib/bgzf.h"
#include "htslib/kstring.h"

/* lines: n_lines SAM lines separated by '\n'.  Writes the records to `tmp_path` through bam_write1 and reads the stream back into out
 * (at most cap bytes).  Returns the number of bytes, -1 - i when line i does not parse, -100000 on an I/O failure. */
long long ref_bam_encode(const char* header_text, const char* lines, const char* tmp_path, uint8_t* out, unsigned long long cap)
{
    bam_hdr_t* h = sam_hdr_parse((int)strlen(header_text), header_text);
    if (!h) return -100000;
    bam1_t* b = bam_init1();
    BGZF* fp = bgzf_open(tmp_path, "wu");
    if (!fp) { bam_destroy1(b); bam_hdr_destroy(h); return -100000; }
    kstring_t s = { 0, 0, NULL };
    long long ret = 0, i = 0;
    const char* p = lines;
    while (*p) {
        const char* e = strchr(p, '\n');
        size_t len = e ? (size_t)(e - p) : strlen(p);
        s.l = 0;
        kputsn(p, len, &s);
        if (sam_parse1(&s, h, b) < 0) { ret = -1 - i; break; }
        if (bam_write1(fp, b) < 0) { ret = -100000; break; }
        ++i;
        p += len + (e ? 1 : 0);
    }
    free(s.s);
    bam_destroy1(b);
    bam_hdr_destroy(h);
    if (bgzf_close(fp) < 0 && ret == 0) ret = -100000;
    if (ret < 0) return ret;
    fp = bgzf_open(tmp_path, "r");
    if (!fp) return -100000;
    ssize_t got = bgzf_read(fp, out, (size_t)cap);
    bgzf_close(fp);
    return got < 0 ? -100000 : (long long)got;
}

/* every record of a .bam file as sam_format1 text, each followed by '\n', into out (at most cap bytes, NUL-terminated).  Returns the
 * number of records, -1 when the file or its header cannot be read, -2 when out is too small. */
long long ref_bam_format(const char* path, char* out, unsigned long long cap)
{
    samFile* fp = sam_open(path, "r");
    if (!fp) return -1;
    bam_hdr_t* h = sam_hdr_read(fp);
    if (!h) { sam_close(fp); return -1; }
    bam1_t* b = bam_init1();
    kstring_t s = { 0, 0, NULL };
    long long n = 0;
    unsigned long long used = 0;
    while (sam_read1(fp, h, b) >= 0) {
        s.l = 0;
        sam_format1(h, b, &s);
        if (used + s.l + 2 > cap) { n = -2; break; }
        memcpy(out + used, s.s, s.l);
        used += s.l;
        out[used++] = '\n';
        ++n;
    }
    if (cap) out[used < cap ? used : cap - 1] = 0;
    free(s.s);
    bam_destroy1(b);
    bam_hdr_destroy(h);
    sam_close(fp);
    return n;
}

int ref_reg2bin(long long beg, long long end) { return hts_reg2bin(beg, end, 14, 5); }
