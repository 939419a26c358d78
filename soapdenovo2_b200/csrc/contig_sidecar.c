/* contig_sidecar.c -- f2 (SURVEY 8f): the `contig` side of the pregraph -> contig hand-over, without the gzip'ed text.
 *
 * The engine can write the edges it builds as a binary sidecar `<prefix>.edge.b200` next to the byte-identical `.edge.gz`
 * (PGB200_EDGE_SIDECAR=1; format: pgb200_edge_sidecar_header in include/pregraph_b200.h).  This file is the reader a maintainer adds to SOAPdenovo2:
 * a `loadEdge()` that fills `edge_array` from the sidecar exactly as the reference's text loader does (loadPreGraph.c:448-544:
 * same allocation, same fields, same buildReverseComplementEdge / createArcMemo / loadPreArcs calls) and falls back to that loader
 * when there is no sidecar.  Nothing of the reference is modified in source: scripts/link_dropin.sh renames the original symbol in
 * the reference's OWN object (`objcopy --redefine-sym loadEdge=loadEdge_text loadPreGraph.o`) and links this file beside it.
 * It is compiled against the reference's headers where they lie (-I$REF/standardPregraph/inc, -DMER63 | -DMER127).
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "stdinc.h"
#include "newhash.h"
#include "kmerhash.h"
#include "extfunc.h"
#include "extvab.h"
#include "../../include/pregraph_b200.h"

extern void loadEdge_text(char *graphfile);                 /* the reference's loadEdge, renamed at link time */
extern void buildReverseComplementEdge(unsigned int edgeno);  /* static in loadPreGraph.c; made global in the object at link time */

/* The reference keeps loadPreArcs / add1Arc static (loadPreGraph.c:30, 580-641, 658-685) and inlines them into its loadEdge, so
 * their logic is restated here: one line of <prefix>.preArc = "from to weight to weight ..."; an arc from->to implies the arc
 * twin(to)->twin(from); existing arcs only gain multiplicity; new arcs are pushed at the head of the edge's list. */
static void sidecar_add_arc(unsigned int from_ed, unsigned int to_ed, unsigned int weight)
{
    unsigned int bal_fe, bal_te;
    ARC *parc, *bal_parc;
    if (edge_array[from_ed].to_vt != edge_array[to_ed].from_vt) return;
    bal_fe = getTwinEdge(from_ed);
    bal_te = getTwinEdge(to_ed);
    if (from_ed > num_ed || to_ed > num_ed || bal_fe > num_ed || bal_te > num_ed) return;
    parc = getArcBetween(from_ed, to_ed);
    if (parc) {
        parc->multiplicity += weight;
        parc->bal_arc->multiplicity += weight;
        return;
    }
    parc = allocateArc(to_ed);
    parc->multiplicity = weight;
    parc->prev = NULL;
    if (edge_array[from_ed].arcs) edge_array[from_ed].arcs->prev = parc;
    parc->next = edge_array[from_ed].arcs;
    edge_array[from_ed].arcs = parc;
    if (bal_te == from_ed) {            /* A -> A': the arc is its own twin */
        parc->bal_arc = parc;
        parc->multiplicity += weight;
        return;
    }
    bal_parc = allocateArc(bal_fe);
    bal_parc->multiplicity = weight;
    bal_parc->prev = NULL;
    if (edge_array[bal_te].arcs) edge_array[bal_te].arcs->prev = bal_parc;
    bal_parc->next = edge_array[bal_te].arcs;
    edge_array[bal_te].arcs = bal_parc;
    parc->bal_arc = bal_parc;
    bal_parc->bal_arc = parc;
}
static void sidecar_load_prearcs(char *graphfile)
{
    char name[512], line[1024], *seg;
    FILE *fp;
    snprintf(name, sizeof name, "%s.preArc", graphfile);
    fp = ckopen(name, "r");
    arcCounter = 0;
    while (fgets(line, sizeof line, fp) != NULL) {
        unsigned int from_ed, target, weight;
        seg = strtok(line, " ");
        from_ed = atoi(seg);
        while ((seg = strtok(NULL, " ")) != NULL) {
            target = atoi(seg);
            seg = strtok(NULL, " ");
            weight = atoi(seg);
            sidecar_add_arc(from_ed, target, weight);
        }
    }
    fprintf(stderr, "%lli pre-arcs loaded.\n", arcCounter);
    fclose(fp);
}

void loadEdge(char *graphfile)
{
    char name[512];
    FILE *fp;
    pgb200_edge_sidecar_header h;
    unsigned long long r;
    int index = -1;
    unsigned int j;
    snprintf(name, sizeof name, "%s.edge.b200", graphfile);
    fp = fopen(name, "rb");
    if (!fp) { loadEdge_text(graphfile); return; }
    if (fread(&h, sizeof h, 1, fp) != 1 || memcmp(h.magic, PGB200_SIDECAR_MAGIC, 8) != 0 || h.version != PGB200_SIDECAR_VERSION || h.kmer_words != sizeof(Kmer) / 8) {
        fprintf(stderr, "%s is not an edge sidecar of this build; reading %s.edge.gz instead.\n", name, graphfile);
        fclose(fp);
        loadEdge_text(graphfile);
        return;
    }
    num_ed_limit = 1.2 * num_ed;
    edge_array = (EDGE *)ckalloc((num_ed_limit + 3) * sizeof(EDGE));
    for (j = num_ed + 1; j <= num_ed_limit; j++) edge_array[j].seq = NULL;
    for (r = 0; r < h.n_records; r++) {
        int rec[4];
        Kmer from_kmer, to_kmer;
        char *tightSeq;
        unsigned int edgeno;
        if (fread(rec, sizeof rec, 1, fp) != 1 || fread(&from_kmer, sizeof(Kmer), 1, fp) != 1 || fread(&to_kmer, sizeof(Kmer), 1, fp) != 1) {
            fprintf(stderr, "%s is truncated.\n", name);
            exit(-1);
        }
        tightSeq = (char *)ckalloc((rec[0] / 4 + 1) * sizeof(char));
        if (fread(tightSeq, 1, (size_t)rec[3], fp) != (size_t)rec[3]) { fprintf(stderr, "%s is truncated.\n", name); exit(-1); }
        index++;
        edgeno = index + 1;
        edge_array[edgeno].length = rec[0];
        edge_array[edgeno].cvg = rec[1];
        edge_array[edgeno].from_vt = kmer2vt(from_kmer);
        edge_array[edgeno].to_vt = kmer2vt(to_kmer);
        edge_array[edgeno].seq = tightSeq;
        edge_array[edgeno].bal_edge = rec[2] + 1;
        edge_array[edgeno].rv = NULL;
        edge_array[edgeno].arcs = NULL;
        edge_array[edgeno].flag = 0;
        edge_array[edgeno].deleted = 0;
        if (rec[2]) {
            buildReverseComplementEdge(edgeno);
            index++;
        }
    }
    fclose(fp);
    fprintf(stderr, "%d edge(s) input.\n", index + 1);
    createArcMemo();
    sidecar_load_prearcs(graphfile);
}
