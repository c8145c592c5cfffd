/*
 * fse_b200_file.c -- the `.fse` frame format on top of libfse_b200 (SURVEY.md section 8f-2).
 *
 * Reads and writes exactly the container of the reference's file tool (programs/fileio.c:121-128,266-626): a file written here
 * is byte-identical to the one `fse -e` / `fse -h` of the reference writes, and either tool decodes the other's output
 * (tests/test_frame_gpu.py checks both against the reference CLI compiled from the unmodified sources).  The layout, the coding
 * parameters and the checksum are the library's: FSEB200_frame_compress_host / FSEB200_frame_decompress_host
 * (include/fse_b200.h) code the whole file in one call each, so this program is file I/O around them.
 *
 * With -m, every input file is one frame of one batch call (FSEB200_frame_{compress,decompress}_host_batch): many small files
 * share the chunk pipeline and the device's checksum kernel instead of paying one call each.
 *
 * usage: fse_b200_file [-e | -h] [-B<id>] <input> <output>      compress (default -e = FSE)
 *        fse_b200_file -d <input> <output>                      decompress (codec from the magic number)
 *        fse_b200_file -m [-e | -h] [-B<id>] <files>...         compress each file to <file>.fse
 *        fse_b200_file -d -m <files>.fse...                     decompress each file to its name without .fse
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

/* the n files as one batch: sizes[f] and each file's bytes back to back */
static unsigned char* read_files(char** names, size_t n, size_t* sizes, size_t* total)
{
    unsigned char* all = NULL;
    size_t f;
    *total = 0;
    for (f = 0; f < n; f++) {
        unsigned char* const p = read_file(names[f], &sizes[f]);
        all = (unsigned char*)realloc(all, *total + sizes[f] + 1);
        if (!all) die("out of memory");
        memcpy(all + *total, p, sizes[f]);
        *total += sizes[f];
        free(p);
    }
    return all;
}

static int compress_files(char** names, size_t n, int codec, unsigned blockId)
{
    size_t* const sizes = (size_t*)malloc((n + 1) * sizeof(size_t));
    size_t* const offsets = (size_t*)malloc((n + 1) * sizeof(size_t));
    size_t* const results = (size_t*)malloc((n + 1) * sizeof(size_t));
    size_t total, cap = 0, f, r;
    unsigned char *src, *frames;
    char* outName;
    if (!sizes || !offsets || !results) die("out of memory");
    src = read_files(names, n, sizes, &total);
    for (f = 0; f < n; f++) cap += FSEB200_frame_compressBound(sizes[f], blockId);
    frames = (unsigned char*)malloc(cap + 1);
    if (!frames) die("out of memory");
    r = FSEB200_frame_compress_host_batch(codec, blockId, n, frames, cap, offsets, results, src, sizes);
    if (FSE_isError(r)) die(FSE_getErrorName(r));
    for (f = 0; f < n; f++) {
        if (FSE_isError(results[f])) { fprintf(stderr, "fse_b200_file: %s: %s\n", names[f], FSE_getErrorName(results[f])); exit(1); }
        outName = (char*)malloc(strlen(names[f]) + 5);
        if (!outName) die("out of memory");
        strcpy(outName, names[f]); strcat(outName, ".fse");
        write_file(outName, frames + offsets[f], results[f]);
        free(outName);
    }
    fprintf(stderr, "Compressed %llu files, %llu bytes into %llu bytes\n", (unsigned long long)n, (unsigned long long)total,
            (unsigned long long)offsets[n]);
    free(frames); free(src); free(results); free(offsets); free(sizes);
    return 0;
}

static int decompress_files(char** names, size_t n)
{
    size_t* const sizes = (size_t*)malloc((n + 1) * sizeof(size_t));
    size_t* const offsets = (size_t*)malloc((n + 1) * sizeof(size_t));
    size_t* const caps = (size_t*)malloc((n + 1) * sizeof(size_t));
    size_t* const results = (size_t*)malloc((n + 1) * sizeof(size_t));
    size_t total, f, r, capTotal = 0, at = 0;
    unsigned char *in, *dst;
    char* outName;
    if (!sizes || !offsets || !caps || !results) die("out of memory");
    for (f = 0; f < n; f++) {
        size_t const len = strlen(names[f]);
        if (len < 5 || strcmp(names[f] + len - 4, ".fse")) { fprintf(stderr, "fse_b200_file: %s: no .fse suffix\n", names[f]); exit(1); }
    }
    in = read_files(names, n, sizes, &total);
    offsets[0] = 0;
    for (f = 0; f < n; f++) {
        size_t const b = FSEB200_frame_decompress_bound(in + offsets[f], sizes[f]);
        if (FSE_isError(b)) { fprintf(stderr, "fse_b200_file: %s: Decoding error : %s\n", names[f], FSE_getErrorName(b)); exit(1); }
        caps[f] = b; capTotal += b;
        offsets[f + 1] = offsets[f] + sizes[f];
    }
    dst = (unsigned char*)malloc(capTotal + 1);
    if (!dst) die("out of memory");
    r = FSEB200_frame_decompress_host_batch(n, dst, caps, results, in, offsets);
    if (FSE_isError(r)) die(FSE_getErrorName(r));
    for (f = 0; f < n; f++) {
        size_t const len = strlen(names[f]);
        if (FSE_isError(results[f])) { fprintf(stderr, "fse_b200_file: %s: Decoding error : %s\n", names[f], FSE_getErrorName(results[f])); exit(1); }
        outName = (char*)malloc(len + 1);
        if (!outName) die("out of memory");
        memcpy(outName, names[f], len - 4); outName[len - 4] = 0;
        write_file(outName, dst + at, results[f]);
        free(outName);
        at += caps[f];
    }
    fprintf(stderr, "Decoded %llu files\n", (unsigned long long)n);
    free(dst); free(in); free(results); free(caps); free(offsets); free(sizes);
    return 0;
}

int main(int argc, char** argv)
{
    int codec = 0, decode = 0, many = 0, i;
    unsigned blockId = 5;                                             /* FIO_BLOCKSIZEID_DEFAULT: 32 KB */
    const char* in = NULL; const char* out = NULL;
    char** files = (char**)malloc((size_t)argc * sizeof(char*));
    size_t nFiles = 0;
    if (!files) die("out of memory");
    for (i = 1; i < argc; i++) {
        if (!strcmp(argv[i], "-e")) codec = 0;
        else if (!strcmp(argv[i], "-h")) codec = 1;
        else if (!strcmp(argv[i], "-d")) decode = 1;
        else if (!strcmp(argv[i], "-m")) many = 1;
        else if (!strncmp(argv[i], "-B", 2)) { blockId = (unsigned)atoi(argv[i] + 2); if (blockId > 6) die("block size id must be 0..6"); }
        else if (many) files[nFiles++] = argv[i];
        else if (!in) in = argv[i];
        else if (!out) out = argv[i];
        else die("too many arguments");
    }
    if (many) {
        if (in) die("-m comes before the file names");
        if (!nFiles) die("usage: fse_b200_file -m [-e|-h] [-B<id>] <files>...  |  fse_b200_file -d -m <files>.fse...");
        return decode ? decompress_files(files, nFiles) : compress_files(files, nFiles, codec, blockId);
    }
    if (!in || !out) die("usage: fse_b200_file [-e|-h] [-B<id>] <in> <out>  |  fse_b200_file -d <in> <out>");
    return decode ? decompress_file(in, out) : compress_file(in, out, codec, blockId);
}
