/* pregraph_shim.c -- the ONE object a maintainer compiles into SOAPdenovo-{63,127}mer in place of pregraph.c (and of the five
 * files only pregraph.c calls into: prlHashReads.c cutTipPreGraph.c node2edge.c prlRead2path.c output_pregraph.c).
 * It provides the symbol the reference's main.c binds (main.c:29 `extern int call_pregraph(int, char **)`, called at main.c:74 for
 * the `pregraph` sub-command and main.c:341 inside `all`) and fixes the 63-mer / 127-mer flavour at BUILD time, exactly as the
 * reference does with -DMER63 / -DMER127 (standardPregraph/Makefile:51-66).  scripts/link_dropin.sh builds both flavours this way.
 *
 * It also keeps the process-level contract of the reference's call_pregraph (pregraph.c:62-139) towards the other stages of `all`:
 *   in :  `all` does not forward -a in argv, it sets the global initKmerSetSize (main.c:202) -- handed on as "-a <n>";
 *   out:  overlaplen (after the odd / 13..63|127 fix-ups), thrd_num, repsTie, deLowKmer stay set; initKmerSetSize is reset to 0
 *         (pregraph.c:122).  The globals are the reference's own (inc/global.h:28,67,71,79,90); they are declared weak so that the
 *         shim also links where they do not exist.
 *
 * call_align (map.c:96; declared main.c:34, called main.c:87 for `map` and main.c:451 inside `all`) runs the GPU map stage,
 * pgb200_map_main, and keeps the reference's contract towards `scaff` (scaffold.c:59-105), which reloads K, the contig lengths and
 * the insert sizes from the files: what survives in globals is what the reference's call_align leaves.
 *   out:  overlaplen = the K map used (K of <prefix>.preGraphBasic, 23 without it, or the -k value), deltaKmer = that K minus -k
 *         when -k applies, smallKmer (-k), thrd_num (-p), fill (-f); contig_array is freed and NULL and num_ctg is the contig count
 *         of <prefix>.ContigIndex when map had to load it (prlRead2Ctg.c:858-861, 1048-1052, basicContigInfo :735-737).
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "../../include/pregraph_b200.h"
#ifndef PGB_FLAVOUR127
#error "compile with -DPGB_FLAVOUR127=0 (SOAPdenovo-63mer) or -DPGB_FLAVOUR127=1 (SOAPdenovo-127mer)"
#endif
extern int initKmerSetSize __attribute__((weak));
extern int overlaplen __attribute__((weak));
extern int thrd_num __attribute__((weak));
extern char repsTie __attribute__((weak));     /* `boolean` is a char, inc/def2.h:25 */
extern char deLowKmer __attribute__((weak));
extern int smallKmer __attribute__((weak));
extern int deltaKmer __attribute__((weak));
extern char fill __attribute__((weak));
extern void *contig_array __attribute__((weak));   /* CONTIG *, inc/global.h:52 */
extern unsigned int num_ctg __attribute__((weak));

int call_pregraph(int argc, char **argv)
{
    char abuf[16];
    char *av[64];
    int n = 0, i, have_a = 0, K = 23, P = 8, R = 0, D = 0, rc;
    for (i = 0; i < argc && n < 60; i++) {
        av[n++] = argv[i];
        if (strncmp(argv[i], "-a", 2) == 0) have_a = 1;
        else if (strcmp(argv[i], "-R") == 0) R = 1;
        else if (i + 1 < argc && strcmp(argv[i], "-K") == 0) K = atoi(argv[i + 1]);
        else if (i + 1 < argc && strcmp(argv[i], "-p") == 0) P = atoi(argv[i + 1]);
        else if (i + 1 < argc && strcmp(argv[i], "-d") == 0) D = atoi(argv[i + 1]) >= 0 ? atoi(argv[i + 1]) : 0;
    }
    if (&initKmerSetSize && initKmerSetSize > 0 && !have_a) {
        snprintf(abuf, sizeof abuf, "%d", initKmerSetSize);
        av[n++] = "-a";
        av[n++] = abuf;
    }
    av[n] = NULL;
    rc = pgb200_pregraph_main(n, av, PGB_FLAVOUR127);
    if (K % 2 == 0) K++;
    if (K < 13) K = 13;
    if (K > (PGB_FLAVOUR127 ? 127 : 63)) K = PGB_FLAVOUR127 ? 127 : 63;
    if (&overlaplen) overlaplen = K;
    if (&thrd_num) thrd_num = P;
    if (&repsTie) repsTie = (char)R;
    if (&deLowKmer) deLowKmer = (char)D;
    if (&initKmerSetSize) initKmerSetSize = 0;
    return rc;
}

static int first_int_after(const char *path, char tag, int skip, int dflt)   /* the value map reads from line `tag...` (map.c:62-72) */
{
    char line[1024];
    int v = dflt, n;
    char ch;
    FILE *fp = fopen(path, "r");
    if (!fp) return dflt;
    while (fgets(line, sizeof line, fp)) {
        if (line[0] != tag) continue;
        if (tag == 'V') { if (sscanf(line + skip, "%d %c %d", &n, &ch, &v) != 3) v = dflt; }
        else if (sscanf(line + skip, "%d", &v) != 1) v = dflt;
        break;
    }
    fclose(fp);
    return v;
}

int call_align(int argc, char **argv)
{
    char path[1024];
    const char *g = NULL;
    int i, K, k = 0, P = 8, F = 0, had_array = &contig_array && contig_array != NULL, rc;
    for (i = 1; i < argc; i++) {
        if (strcmp(argv[i], "-f") == 0) F = 1;
        else if (i + 1 < argc && strcmp(argv[i], "-g") == 0) g = argv[i + 1];
        else if (i + 1 < argc && strcmp(argv[i], "-k") == 0) k = atoi(argv[i + 1]);
        else if (i + 1 < argc && strcmp(argv[i], "-p") == 0) P = atoi(argv[i + 1]);
    }
    rc = pgb200_map_main(argc, argv, PGB_FLAVOUR127);   /* ends the process on any error, as the reference does */
    snprintf(path, sizeof path, "%s.preGraphBasic", g ? g : "");
    K = first_int_after(path, 'V', 6, 23);
    if (k > 12 && k <= (PGB_FLAVOUR127 ? 127 : 63) && k % 2 == 1) {
        if (&deltaKmer) deltaKmer = K - k;
        K = k;
    }
    if (&overlaplen) overlaplen = K;
    if (&smallKmer) smallKmer = k;
    if (&thrd_num) thrd_num = P;
    if (F && &fill) fill = 1;
    if (had_array) { free(contig_array); contig_array = NULL; }
    else if (&num_ctg) {
        snprintf(path, sizeof path, "%s.ContigIndex", g ? g : "");
        num_ctg = (unsigned int)first_int_after(path, 'E', 8, (int)num_ctg);
    }
    return rc;
}
