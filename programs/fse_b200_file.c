/*
 * fse_b200_file.c -- the `.fse` frame format on top of libfse_b200 (SURVEY.md section 8f-2).
 *
 * Reads and writes exactly the container of the reference's file tool (programs/fileio.c:121-128,266-626): a file written here
 * is byte-identical to the one `fse -e` / `fse -h` of the reference writes, and either tool decodes the other's output
 * (tests/test_frame_gpu.py checks both against the reference CLI compiled from the unmodified sources).  The layout, the coding
 * parameters and the checksum are the library's: FSEB200_frame_compress_host / FSEB200_frame_decompress_host
 * (include/fse_b200.h) code the whole file in one call each, so this program is file I/O around them.
 *
 * usage: fse_b200_file [-e | -h] [-B<id>] <input> <output>      compress (default -e = FSE)
 *        fse_b200_file -d <input> <output>                      decompress (codec from the magic number)
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "fse_b200.h"

static void die(const char* what)
{
    fprintf(stderr, "fse_b200_file: %s\n", what);
    exit(1);
}

static unsigned char* read_file(const char* name, size_t* size)
{
    FILE* f = fopen(name, "rb");
    unsigned char* buf;
    long n;
    if (!f) die("cannot open input");
    if (fseek(f, 0, SEEK_END) != 0 || (n = ftell(f)) < 0 || fseek(f, 0, SEEK_SET) != 0) die("cannot size input");
    buf = (unsigned char*)malloc((size_t)n + 1);
    if (!buf) die("out of memory");
    if (n && fread(buf, 1, (size_t)n, f) != (size_t)n) die("read error");
    fclose(f);
    *size = (size_t)n;
    return buf;
}

static void write_file(const char* name, const void* p, size_t n)
{
    FILE* f = fopen(name, "wb");
    if (!f) die("cannot open output");
    if (n && fwrite(p, 1, n, f) != n) die("write error");
    if (fclose(f) != 0) die("write error");
}

static int compress_file(const char* in, const char* out, int codec, unsigned blockId)
{
    size_t n, cap, r;
    unsigned char* const src = read_file(in, &n);
    unsigned char* frame;
    cap = FSEB200_frame_compressBound(n, blockId);
    if (FSE_isError(cap)) die(FSE_getErrorName(cap));
    frame = (unsigned char*)malloc(cap);
    if (!frame) die("out of memory");
    r = FSEB200_frame_compress_host(codec, blockId, frame, cap, src, n);
    if (FSE_isError(r)) die(FSE_getErrorName(r));
    write_file(out, frame, r);
    fprintf(stderr, "Compressed %llu bytes into %llu bytes ==> %.2f%%\n", (unsigned long long)n, (unsigned long long)r,
            n ? 100.0 * (double)r / (double)n : 0.0);
    free(frame); free(src);
    return 0;
}

static int decompress_file(const char* in, const char* out)
{
    size_t n, bound, r;
    unsigned char* const frame = read_file(in, &n);
    unsigned char* dst;
    bound = FSEB200_frame_decompress_bound(frame, n);
    if (FSE_isError(bound)) die(FSE_getErrorName(bound));
    dst = (unsigned char*)malloc(bound + 1);
    if (!dst) die("out of memory");
    r = FSEB200_frame_decompress_host(dst, bound, frame, n);
    if (FSE_isError(r)) { fprintf(stderr, "fse_b200_file: Decoding error : %s\n", FSE_getErrorName(r)); exit(1); }
    write_file(out, dst, r);
    fprintf(stderr, "Decoded %llu bytes\n", (unsigned long long)r);
    free(dst); free(frame);
    return 0;
}

int main(int argc, char** argv)
{
    int codec = 0, decode = 0, i;
    unsigned blockId = 5;                                             /* FIO_BLOCKSIZEID_DEFAULT: 32 KB */
    const char* in = NULL; const char* out = NULL;
    for (i = 1; i < argc; i++) {
        if (!strcmp(argv[i], "-e")) codec = 0;
        else if (!strcmp(argv[i], "-h")) codec = 1;
        else if (!strcmp(argv[i], "-d")) decode = 1;
        else if (!strncmp(argv[i], "-B", 2)) { blockId = (unsigned)atoi(argv[i] + 2); if (blockId > 6) die("block size id must be 0..6"); }
        else if (!in) in = argv[i];
        else if (!out) out = argv[i];
        else die("too many arguments");
    }
    if (!in || !out) die("usage: fse_b200_file [-e|-h] [-B<id>] <in> <out>  |  fse_b200_file -d <in> <out>");
    return decode ? decompress_file(in, out) : compress_file(in, out, codec, blockId);
}
