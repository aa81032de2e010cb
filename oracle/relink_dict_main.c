/* relink_dict_main.c -- TEST INFRASTRUCTURE.  The reference's frame DECODER over our dictionary decoding: oracle/relink_dict.mk
 * compiles the UNMODIFIED lib/lizard_frame.c + lib/xxhash/xxhash.c from the reference tree together with this file and links
 * the result against liblizard_b200.so.  A frame of linked blocks makes the frame layer call Lizard_decompress_safe_usingDict
 * for every block after the first (lib/lizard_frame.c:1148-1157 straight into the caller's buffer, with the previous output as
 * an in-place prefix; :1176-1197 through its temporary buffer, with an external dictionary), so this program decodes such a
 * frame with our library doing every block.
 *
 *   relinked_dict <frame-in> <out-path> <dst-chunk>
 *   Feeds the whole frame and takes the output `dst-chunk` bytes per LizardF_decompress call (a chunk below the block size
 *   sends the blocks through the frame layer's temporary buffer), then writes the output to out-path and nothing else.
 *   exit 0 = frame decoded, 1 = a call failed
 */
#include <stdio.h>
#include <stdlib.h>
#include "lizard_frame.h"          /* the reference's header (-I$(REF)/lib) */

int main(int argc, char** argv)
{
    if (argc < 4) { fprintf(stderr, "usage: %s frame-in out dst-chunk\n", argv[0]); return 1; }
    const size_t chunk = (size_t)atol(argv[3]);
    FILE* f = fopen(argv[1], "rb");
    if (!f || chunk == 0) return 1;
    fseek(f, 0, SEEK_END);
    const size_t fsize = (size_t)ftell(f);
    fseek(f, 0, SEEK_SET);
    char* frame = (char*)malloc(fsize + 1);
    if (!frame || fread(frame, 1, fsize, f) != fsize) return 1;
    fclose(f);

    LizardF_decompressionContext_t d;
    if (LizardF_isError(LizardF_createDecompressionContext(&d, LIZARDF_VERSION))) return 1;
    size_t cap = 1 << 20, op = 0, ip = 0, hint = 1;
    char* out = (char*)malloc(cap);
    while (hint != 0) {
        if (op + chunk > cap) { cap = 2 * (op + chunk); out = (char*)realloc(out, cap); if (!out) return 1; }
        size_t si = fsize - ip, so = chunk;
        hint = LizardF_decompress(d, out + op, &so, frame + ip, &si, NULL);
        if (LizardF_isError(hint)) { fprintf(stderr, "LizardF_decompress: %s\n", LizardF_getErrorName(hint)); return 1; }
        ip += si; op += so;
        if (si == 0 && so == 0) break;
    }
    LizardF_freeDecompressionContext(d);
    f = fopen(argv[2], "wb");
    if (!f || fwrite(out, 1, op, f) != op || fclose(f) != 0) return 1;
    return hint == 0 ? 0 : 1;
}
