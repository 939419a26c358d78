/* main.c -- CLI front end: `pregraph-b200-63mer pregraph -s cfg -K k -p P [-a G] [-d D] [-R] -o prefix` and
 * `pregraph-b200-63mer map -s cfg -g prefix [-f] [-p n] [-k k]` (same sub-command dispatch shape as the reference's main.c:59-104).  Host orchestration stays in C/C++;
 * everything k-mer shaped runs on the GPU inside libpregraph_b200.so. */
#include <stdio.h>
#include <string.h>
#include "../../include/pregraph_b200.h"

#ifndef PGB_FLAVOUR127
#define PGB_FLAVOUR127 0
#endif

int main(int argc, char **argv)
{
    if (argc == 4 && strcmp(argv[1], "edgegz") == 0 && strcmp(argv[2], "-g") == 0) {
        /* host only: <prefix>.edge.b200 -> the byte-identical <prefix>.edge.gz (after a stage run with PGB200_EDGE_SIDECAR=only) */
        if (pgb200_sidecar_to_edge_gz(argv[3])) { fprintf(stderr, "%s\n", pgb200_last_error()); return 1; }
        return 0;
    }
    if (argc >= 2 && strcmp(argv[1], "map") == 0) return pgb200_map_main(argc - 1, argv + 1, PGB_FLAVOUR127);
    if (argc < 2 || strcmp(argv[1], "pregraph") != 0) {
        fprintf(stderr, "Usage: %s pregraph -s configFile -o outputGraph [-R] [-K kmer -p P -a G -d D]\n"
                        "       %s map -s configFile -g inputGraph [-f] [-p n_cpu -k kmer_R2C]\n"
                        "       %s edgegz -g outputGraph      (edge sidecar -> .edge.gz, host only)\n"
                        "(the GPU engine replaces the pregraph and map stages; contig/scaff stay with SOAPdenovo-%s)\n",
                argv[0], argv[0], argv[0], PGB_FLAVOUR127 ? "127mer" : "63mer");
        return 1;
    }
    return pgb200_pregraph_main(argc - 1, argv + 1, PGB_FLAVOUR127);
}
