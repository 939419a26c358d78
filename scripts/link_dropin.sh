#!/bin/bash
# Link-level drop-in check (INTEGRATION.md section 1): the reference's OWN objects (oracle/_ref/o{63,127}/*.o, compiled unmodified
# from /root/reference by oracle/Makefile) minus the six files the engine replaces, plus pregraph_shim.o and libpregraph_b200.so.
# The result, oracle/_ref/SOAPdenovo-{63,127}mer-b200, is the reference's main() / contig / scaff around the GPU pregraph and the
# GPU map (map.o, prlHashCtg.o and prlRead2Ctg.o are left out: nothing else uses their symbols; the shim's call_align replaces them):
#   SOAPdenovo-63mer-b200 pregraph ... | contig ... | map ... | all ...   (tests/test_gpu_dropin.py, tests/test_gpu_map_dropin.py compare
#   them with the unmodified binary)
# f2: the same binaries read the engine's binary edge sidecar (<prefix>.edge.b200) when there is one -- csrc/contig_sidecar.c is linked
# beside the reference's loadPreGraph.o, whose loadEdge symbol is renamed (and whose static buildReverseComplementEdge is made global)
# IN THE OBJECT with objcopy; no reference source is touched or copied.
set -e
cd "$(dirname "$0")/.."
REF=oracle/_ref
LIB=soapdenovo2_b200/lib
REFSRC=${REFSRC:-/root/reference}
[ -f $LIB/libpregraph_b200.so ] || make -s -j8 -C soapdenovo2_b200/csrc
if [ ! -d $REFSRC/standardPregraph/inc ]; then
  echo "link_dropin: $REFSRC absent (GPU box): keeping the prebuilt $REF/SOAPdenovo-*mer-b200"; exit 0
fi
for fl in 63 127; do
  [ -d $REF/o$fl ] || { echo "link_dropin: $REF/o$fl missing (run make -C oracle ref where /root/reference exists)"; exit 2; }
  T=$REF/o$fl/.b200_tmp; rm -rf $T; mkdir -p $T
  objs=$(ls $REF/o$fl/*.o | grep -v -E '/(pregraph|prlHashReads|cutTipPreGraph|node2edge|prlRead2path|output_pregraph|loadPreGraph|map|prlHashCtg|prlRead2Ctg)\.o$')
  gcc -O2 -c -DPGB_FLAVOUR127=$([ $fl = 127 ] && echo 1 || echo 0) soapdenovo2_b200/csrc/pregraph_shim.c -o $T/pregraph_shim.o
  objcopy --redefine-sym loadEdge=loadEdge_text --globalize-symbol=buildReverseComplementEdge $REF/o$fl/loadPreGraph.o $T/loadPreGraph_renamed.o
  gcc -O2 -w -fcommon -c -DMER$fl -I$REFSRC/standardPregraph/inc soapdenovo2_b200/csrc/contig_sidecar.c -o $T/contig_sidecar.o
  # libbam.a (b= inputs of the other stages) ships with the reference; it travels to the GPU box inside the already linked binary
  g++ -no-pie $objs $T/pregraph_shim.o $T/loadPreGraph_renamed.o $T/contig_sidecar.o -L$REFSRC/sparsePregraph/inc -L$LIB -lpregraph_b200 \
      -Wl,-rpath,'$ORIGIN/../../soapdenovo2_b200/lib' -pthread -lz -lm -lbam -lrt -o $REF/SOAPdenovo-${fl}mer-b200
  rm -rf $T
  echo "linked $REF/SOAPdenovo-${fl}mer-b200"
done
