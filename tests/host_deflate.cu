// CPU driver for soapdenovo2_b200/csrc/deflate.cuh: runs the __host__ __device__ pieces one after another (hash chains, match
// search, the lazy automaton, block cuts, tree build, block-type choice, the bit-offset maps, CRC combine) and writes a gzip file.
// tests/test_deflate_host.py compares each file with zlib.compressobj(6, DEFLATED, 31).
//
// usage: host_deflate <in> <out> [<in> <out> ...]; prints one line per file:
//   <in> bytes=.. syms=.. blocks=.. stored=.. fixed=.. dyn=.. maxlen=.. toofar=.. reduced=.. crc_ok=1 off_ok=1
#pragma nv_diag_suppress 20011   // the host-only bit writer passed to the __host__ __device__ tree writers
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <vector>

#include "../soapdenovo2_b200/csrc/deflate.cuh"

using namespace gz;

struct Bits {
    std::vector<u8> out;
    u64 acc = 0;
    int n = 0;
    u64 total = 0;
    void operator()(u32 v, int len) {
        acc |= (u64)v << n;
        n += len;
        total += len;
        while (n >= 8) { out.push_back((u8)acc); acc >>= 8; n -= 8; }
    }
    void align() { if (n) { out.push_back((u8)acc); acc = 0; total += 8 - n; n = 0; } }
};

int main(int argc, char** argv) {
    u32 table[256];
    for (u32 i = 0; i < 256; i++) table[i] = crc_table_entry(i);
    int bad = 0;
    for (int a = 1; a + 1 < argc; a += 2) {
        FILE* f = fopen(argv[a], "rb");
        if (!f) { perror(argv[a]); return 2; }
        std::vector<u8> in;
        u8 buf[1 << 16];
        size_t r;
        while ((r = fread(buf, 1, sizeof buf, f)) > 0) in.insert(in.end(), buf, buf + r);
        fclose(f);
        const i64 N = (i64)in.size();

        // hash chains: distance to the previous position with the same hash (0: none within 32767)
        std::vector<u16> pv(N + 1, 0);
        std::vector<i64> head(1 << 15, -1);
        for (i64 p = 0; p + 2 < N; p++) {
            const u32 h = hash3(in[p], in[p + 1], in[p + 2]);
            if (head[h] >= 0 && p - head[h] < 32768) pv[p] = (u16)(p - head[h]);
            head[h] = p;
        }
        auto B = [&](i64 i) { return in[i]; };
        auto P = [&](i64 i) { return (u32)pv[i]; };

        // the lazy automaton over every loop top, then the terminal one at N
        std::vector<Sym> syms;
        LazyState st = fresh_state();
        int maxlen = 0, toofar = 0, reduced = 0;
        i64 s = 0;
        while (s < N) {
            const i64 base = (i64)slide_base((u64)s, (u64)N, true);
            const Match m = find_match(B, P, s, N - s, base);
            if (m.len128 != m.len32 || m.dist128 != m.dist32) reduced++;   // the quarter chain would answer differently
            bool emit;
            u32 sym;
            i64 pos;
            const i64 nx = lazy_step(st, s, m, s ? in[s - 1] : 0, emit, sym, pos);
            if (emit) {
                syms.push_back(Sym{sym, (u32)pos, 0});
                if ((int)sym_len(sym) > maxlen) maxlen = (int)sym_len(sym);
            }
            s = nx;
        }
        bool term_lit = false;
        if (st.ma) { syms.push_back(Sym{sym_lit(in[N - 1]), (u32)(N - 1), 0}); term_lit = true; }
        for (i64 p = 0; p + 2 < N; p++) {   // positions whose only candidate is a length-3 match beyond TOO_FAR
            const u32 d = pv[p];
            if (d > TOO_FAR && d <= MAX_DIST && p + 3 < N && in[p - d + 3] != in[p + 3] && in[p - d] == in[p] && in[p - d + 1] == in[p + 1]) toofar++;
        }

        // blocks of 16383 symbols; the last block holds the rest (an empty last block when an in-loop flush used the final symbol)
        const u64 T = syms.size();
        u64 nblocks = T / SYM_END + ((T % SYM_END) != 0);
        if (T % SYM_END == 0 && !term_lit) nblocks++;
        Bits bw;
        const u8 hdr[10] = {0x1f, 0x8b, 8, 0, 0, 0, 0, 0, 0, 3};
        for (u8 c : hdr) bw(c, 8);
        OffMap acc = off_plain(0);
        const u64 off0 = bw.total;
        int nst = 0, nfx = 0, ndy = 0;
        BlockTrees* t = new BlockTrees;
        u32 lcode[L_CODES], dcode[D_CODES];
        bool off_ok = true;
        for (u64 k = 0; k < nblocks; k++) {
            const u64 a0 = k * SYM_END, a1 = (k + 1) * SYM_END < T ? (k + 1) * SYM_END : T;
            const bool last = k + 1 == nblocks;
            memset(t->l.freq, 0, sizeof t->l.freq);
            memset(t->d.freq, 0, sizeof t->d.freq);
            for (u64 j = a0; j < a1; j++) {
                const u32 v = syms[j].sym;
                if (!sym_is_match(v)) t->l.freq[v]++;
                else { t->l.freq[257 + length_code((int)sym_len(v) - 3)]++; t->d.freq[dist_code((int)sym_dist(v) - 1)]++; }
            }
            t->l.freq[END_BLOCK] = 1;
            const u64 first = a1 > a0 ? syms[a0].pos : (u64)N;
            const u64 end = last ? (u64)N : syms[a1 - 1].pos + sym_len(syms[a1 - 1].sym);
            const u64 flush_top = last ? (u64)N : syms[a1 - 1].pos + 1;
            const bool stored_ok = first >= slide_base(flush_top, (u64)N, true);
            u64 nbits = 0;
            const int type = plan_block(*t, end - first, stored_ok, &nbits);
            const u64 before = bw.total;
            OffMap m;
            if (type == BT_STORED) {
                nst++;
                bw((u32)last, 3);
                bw.align();
                const u32 len = (u32)(end - first);
                bw(len & 0xffff, 16);
                bw(~len & 0xffff, 16);
                for (u64 i = first; i < end; i++) bw(in[i], 8);
                m = off_stored(len);
            } else {
                (type == BT_FIXED ? nfx : ndy)++;
                bw((u32)(type << 1 | last), 3);
                if (type == BT_DYN) send_all_trees(*t, bw);
                code_tables(*t, type, lcode, dcode);
                for (u64 j = a0; j < a1; j++) send_symbol(syms[j].sym, lcode, dcode, bw);
                bw(lcode[END_BLOCK] & 0xffff, lcode[END_BLOCK] >> 16);
                if (bw.total - before != nbits) off_ok = false;   // plan_block's size is the size written
                m = off_plain(nbits);
            }
            // the composed map of all blocks so far must land where the writer is
            acc = off_then(acc, m);
            if (off_apply(acc, off0) != bw.total) off_ok = false;
        }
        bw.align();
        delete t;

        // CRC: whole, and combined from pieces of varying sizes
        const u32 crc = ~crc_update(~0u, table, in.data(), in.size());
        u32 comb = 0;
        u64 at = 0, step = 1;
        while (at < in.size()) {
            const u64 len = step < in.size() - at ? step : in.size() - at;
            const u32 c = ~crc_update(~0u, table, in.data() + at, len);
            comb = at == 0 ? c : crc_combine(comb, c, len);
            at += len;
            step = step * 3 + 7;
        }
        const bool crc_ok = in.empty() ? crc == 0 : comb == crc;
        for (int i = 0; i < 4; i++) bw((crc >> (8 * i)) & 0xff, 8);
        for (int i = 0; i < 4; i++) bw(((u32)N >> (8 * i)) & 0xff, 8);
        FILE* o = fopen(argv[a + 1], "wb");
        fwrite(bw.out.data(), 1, bw.out.size(), o);
        fclose(o);
        printf("%s bytes=%lld syms=%llu blocks=%llu stored=%d fixed=%d dyn=%d maxlen=%d toofar=%d reduced=%d crc_ok=%d off_ok=%d\n",
               argv[a], (long long)N, (unsigned long long)T, (unsigned long long)nblocks, nst, nfx, ndy, maxlen, toofar, reduced,
               (int)crc_ok, (int)off_ok);
        bad += !crc_ok || !off_ok;
    }
    return bad ? 1 : 0;
}
