/* tests/host_decode.cpp — TEST INFRASTRUCTURE.  A CPU driver around the host+device functions of
 * zstd_b200/csrc/zb_decode_core.cuh: the same header walk, table builders and bitstream readers the CUDA decompressor
 * runs per warp are run here block after block, so that they can be checked against frames of the reference encoder
 * (and of this repo's oracle) in the CPU test suite.  Built by tests/test_host_decode.py with g++; nothing in the
 * product links against it.
 *   size_t zbh_decompress(void* dst, size_t cap, const void* src, size_t size)  -> bytes written, or (size_t)-code
 *   size_t zbh_decompress_usingDict(dst, cap, src, size, dict, dictSize)
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <vector>
#include "../zstd_b200/csrc/zb_decode_core.cuh"

#define ERR(c) ((size_t)-(long)(c))

struct BlockOut { std::vector<u8> lits; std::vector<u64> seqs; u32 sumLL, sumML; ZbdRep transfer; };
/* dependency statistics of the last call (development: how parallel is the match stage of a frame?) */
extern "C" { unsigned long long zbh_nbMatches, zbh_maxDepth, zbh_nearDeps, zbh_anyDeps, zbh_tileDepth; }
static std::vector<unsigned> g_tDepth;
/* which check refused the last call, where the reference decoder's one-shot call may accept: 1 = the end of a Huffman
 * stream of the literals (the reference accepts some streams that read past their start), 2 = a compressed block that
 * regenerates more than Block_Maximum_Size (the reference's one-shot call accepts up to ~32 bytes more) */
extern "C" { unsigned zbh_refusedBy; }

static std::vector<unsigned long long> g_mStart, g_mEnd; static std::vector<unsigned> g_mDepth;
static const u8* g_dict = NULL;            /* the call's dictionary (single-threaded test code) */
static ZbdDictInfo g_di;

/* Huffman decoding table of block b's literals */
static u32 buildHuf(std::vector<u16>& table, u32* logOut, u32* descBytes, const u8* in, const std::vector<ZbdBlock>& B, const ZbdBlock& b)
{
    u8 weights[256]; u32 nbSym = 0, log = 0, len = 0; u32 fse[64]; short norm[16]; u16 next[16];
    const u8* const p = zbd_hufDescription(&b, B.data(), in, g_dict, &g_di, &len);
    u32 const used = zbd_readHufWeights(weights, &nbSym, &log, p, len, fse, norm, next);
    if (!used) return ZBD_CORRUPT;
    u16 start[256];
    zbd_hufStarts(start, weights, nbSym, log);
    table.assign((size_t)1 << log, 0);
    for (u32 s = 0; s < nbSym; s++) zbd_hufFill(table.data(), s, start[s], weights[s], log, 0, 1);
    *logOut = log; *descBytes = used;
    return ZBD_OK;
}

static u32 decodeLiterals(BlockOut& o, const u8* in, const std::vector<ZbdBlock>& B, u32 bi)
{
    const ZbdBlock& b = B[bi];
    const u8* const c = in + b.srcOff;
    o.lits.assign(b.litRegen + 8, 0);
    if (b.litType == 0) { memcpy(o.lits.data(), c + b.litHdr, b.litRegen); return ZBD_OK; }
    if (b.litType == 1) { memset(o.lits.data(), c[b.litHdr], b.litRegen); return ZBD_OK; }
    std::vector<u16> table; u32 log = 0, desc = 0;
    if (buildHuf(table, &log, &desc, in, B, b)) return ZBD_CORRUPT;
    if (b.litType == 3) desc = 0;                               /* treeless: the streams start right behind the header */
    if (desc > b.litComp) return ZBD_CORRUPT;
    const u8* s = c + b.litHdr + desc;
    u32 const total = b.litComp - desc;
    if (b.litStreams == 1) {
        if (zbd_hufDecodeStream(o.lits.data(), b.litRegen, s, total, table.data(), log)) { zbh_refusedBy = 1; return ZBD_CORRUPT; }
        return ZBD_OK;
    }
    u32 off[4], size[4], count[4];
    if (zbd_litStreams(off, size, count, s, total, b.litRegen)) return ZBD_CORRUPT;
    for (u32 k = 0; k < 4; k++)
        if (zbd_hufDecodeStream(o.lits.data() + k * count[0], count[k], s + off[k], size[k], table.data(), log)) { zbh_refusedBy = 1; return ZBD_CORRUPT; }
    return ZBD_OK;
}

static u32 decodeSeqs(BlockOut& o, const u8* in, const std::vector<ZbdBlock>& B, u32 bi)
{
    const ZbdBlock& b = B[bi];
    o.sumLL = o.sumML = 0;
    o.transfer.r[0] = ZBD_SYM(0u, 0u); o.transfer.r[1] = ZBD_SYM(1u, 0u); o.transfer.r[2] = ZBD_SYM(2u, 0u);
    o.seqs.assign(b.nbSeq, 0);
    if (!b.nbSeq) return ZBD_OK;
    u32 T[3][512]; int logs[3]; short norm[64]; u16 next[64];
    for (u32 s = 0; s < 3; s++) if ((logs[s] = zbd_seqTable(T[s], norm, next, s, &b, B.data(), in, g_dict, &g_di)) < 0) return ZBD_CORRUPT;
    const u8* const sec = in + b.srcOff + b.seqOff;
    u32 const avail = b.cSize - b.seqOff;
    u32 desc[3], bitstream;
    if (zbd_locateDescriptions(&b, sec, avail, desc, &bitstream, norm)) return ZBD_CORRUPT;
    return zbd_decodeSequences(o.seqs.data(), b.nbSeq, sec + bitstream, avail - bitstream, T[0], logs[0], T[1], logs[1],
                               T[2], logs[2], &o.sumLL, &o.sumML, &o.transfer);
}

extern "C" size_t zbh_decompress_usingDict(void* dstv, size_t cap, const void* srcv, size_t size, const void* dictv, size_t dictSize)
{
    const u8* const in = (const u8*)srcv;
    u8* const dst = (u8*)dstv;
    g_dict = (const u8*)dictv; memset(&g_di, 0, sizeof(g_di)); zbh_refusedBy = 0;
    if (g_dict && dictSize) { u32 const de = zbd_parseDict(&g_di, g_dict, dictSize); if (de) return ERR(de); }
    const u8* const content = g_dict ? g_dict + g_di.contentOff : NULL;
    size_t const contentSize = g_dict ? dictSize - g_di.contentOff : 0;
    u32 nb = 0, nf = 0;
    u64 litBytes = 0, seqCount = 0;
    u32 e = zbd_walk(in, size, NULL, 0, NULL, 0, &nb, &nf, &litBytes, &seqCount, g_di.entropy != 0, g_di.dictID);
    if (e) return ERR(e);
    std::vector<ZbdBlock> B(nb ? nb : 1); std::vector<ZbdFrame> F(nf ? nf : 1);
    e = zbd_walk(in, size, B.data(), nb, F.data(), nf, &nb, &nf, &litBytes, &seqCount, g_di.entropy != 0, g_di.dictID);
    if (e) return ERR(e);
    size_t out = 0;
    zbh_nbMatches = zbh_maxDepth = zbh_nearDeps = zbh_anyDeps = zbh_tileDepth = 0; g_mStart.clear(); g_mEnd.clear(); g_mDepth.clear(); g_tDepth.clear();
    for (u32 f = 0; f < nf; f++) {
        size_t const frameStart = out;
        ZbdRep rep; rep.r[0] = 1; rep.r[1] = 4; rep.r[2] = 8;
        if (g_di.entropy) { rep.r[0] = g_di.rep[0]; rep.r[1] = g_di.rep[1]; rep.r[2] = g_di.rep[2]; }
        for (u32 bi = F[f].firstBlock; bi < F[f].firstBlock + F[f].nbBlocks; bi++) {
            const ZbdBlock& b = B[bi];
            if (b.type == ZB_BT_RAW) { if (out + b.rawSize > cap) return ERR(70); memcpy(dst + out, in + b.srcOff, b.rawSize); out += b.rawSize; continue; }
            if (b.type == ZB_BT_RLE) { if (out + b.rawSize > cap) return ERR(70); memset(dst + out, in[b.srcOff], b.rawSize); out += b.rawSize; continue; }
            BlockOut o;
            if (decodeLiterals(o, in, B, bi)) return ERR(ZBD_CORRUPT);
            {   u32 const se = decodeSeqs(o, in, B, bi); if (se) return ERR(se); }          /* 20, or 16 for an offset beyond 28 bits */
            if (o.sumLL > b.litRegen) return ERR(ZBD_CORRUPT);
            size_t const regen = (size_t)b.litRegen + o.sumML;
            if (regen > b.blockMax) { zbh_refusedBy = 2; return ERR(ZBD_CORRUPT); }
            if (out + regen > cap) return ERR(70);
            /* the history at the block's end, first as the transfer function says, then by executing: both must agree */
            ZbdRep predicted; for (int k = 0; k < 3; k++) predicted.r[k] = zbd_rep_resolve(o.transfer.r[k], &rep);
            u32 lp = 0;
            for (u32 i = 0; i < b.nbSeq; i++) {
                u64 const q = o.seqs[i];
                u32 const ll = ZBD_SEQ_LL(q), ml = ZBD_SEQ_ML(q);
                u32 const off = zbd_rep_apply(&rep, ZBD_SEQ_OFF(q), ll, false);
                memcpy(dst + out, o.lits.data() + lp, ll); out += ll; lp += ll;
                size_t const inFrame = out - frameStart;
                if (off == 0 || off > inFrame + contentSize) return ERR(ZBD_CORRUPT);
                if (ml && off <= inFrame) {                        /* which earlier matches wrote [src, src + min(ml, off))? */
                    unsigned long long const ss = out - off, se = ss + (ml < off ? ml : off);
                    size_t lo = 0, hi = g_mStart.size();
                    while (lo < hi) { size_t const mid = (lo + hi) / 2; if (g_mEnd[mid] <= ss) lo = mid + 1; else hi = mid; }
                    unsigned depth = 0; bool any = false, near = false;
                    for (size_t j = lo; j < g_mStart.size() && g_mStart[j] < se; j++) { any = true; if (g_mDepth[j] > depth) depth = g_mDepth[j]; if (g_mStart.size() - j <= 32) near = true; }
                    {   /* the kernel's conservative rule: every match from "first one ending behind the tile of ss" to "first one ending behind the first tile at or past se" */
                        size_t a = 0, bnd = g_mStart.size(), c = 0, dnd = g_mStart.size();
                        unsigned long long const t0 = (ss >> 6) << 6, t1 = ((se + 63) >> 6) << 6;
                        while (a < bnd) { size_t const mid = (a + bnd) / 2; if (g_mEnd[mid] <= t0) a = mid + 1; else bnd = mid; }
                        while (c < dnd) { size_t const mid = (c + dnd) / 2; if (g_mEnd[mid] <= t1) c = mid + 1; else dnd = mid; }
                        unsigned dt = 0;
                        for (size_t j = a; j <= c && j < g_mStart.size(); j++) if (g_tDepth[j] > dt) dt = g_tDepth[j];
                        g_tDepth.push_back(dt + 1); if (dt + 1 > zbh_tileDepth) zbh_tileDepth = dt + 1;
                    }
                    g_mStart.push_back(out); g_mEnd.push_back(out + ml); g_mDepth.push_back(depth + 1);
                    zbh_nbMatches++; if (any) zbh_anyDeps++; if (near) zbh_nearDeps++; if (depth + 1 > zbh_maxDepth) zbh_maxDepth = depth + 1;
                }
                for (u32 k = 0; k < ml; k++) {                      /* the gather form the kernel uses; positions in front of the frame are dictionary content */
                    long long const sp = (long long)inFrame - (long long)off + (long long)(k % off);
                    dst[out + k] = sp < 0 ? content[(long long)contentSize + sp] : dst[frameStart + sp];
                }
                out += ml;
            }
            memcpy(dst + out, o.lits.data() + lp, b.litRegen - lp); out += b.litRegen - lp;
            for (int k = 0; k < 3; k++) if (predicted.r[k] != rep.r[k]) return ERR(1);
        }
        if (F[f].contentSize != ZBD_CONTENTSIZE_UNKNOWN && out - frameStart != F[f].contentSize) return ERR(ZBD_CORRUPT);
    }
    return out;
}
extern "C" size_t zbh_decompress(void* dst, size_t cap, const void* src, size_t size) { return zbh_decompress_usingDict(dst, cap, src, size, NULL, 0); }

#ifdef ZBH_CORPUS_MAIN
/* A program over a corpus of inputs, for runs under sanitizers (tests/test_decode_invalid.py): stdin holds records
 * u64 cap, u64 dictSize, dict, u64 size, src (little-endian); stdout gets one line per record: the return value, the
 * sum of out[i] * (i + 1) mod 2^64 over the output, and whether the 16 bytes behind dst[cap) kept their value. */
#include <stdio.h>
static bool readAll(void* p, size_t n) { return fread(p, 1, n, stdin) == n; }
int main()
{
    unsigned long long cap, dn, sn;
    while (readAll(&cap, 8)) {
        std::vector<u8> d, s, out(cap + 16, 0xA5);
        if (!readAll(&dn, 8)) return 2;
        d.resize(dn); if (dn && !readAll(d.data(), dn)) return 2;
        if (!readAll(&sn, 8)) return 2;
        s.resize(sn); if (sn && !readAll(s.data(), sn)) return 2;
        size_t const r = zbh_decompress_usingDict(out.data(), cap, s.data(), sn, dn ? d.data() : NULL, dn);
        unsigned long long h = 0;
        if (r <= cap) for (size_t i = 0; i < r; i++) h += (unsigned long long)out[i] * (i + 1);
        bool guard = true;
        for (size_t i = 0; i < 16; i++) guard = guard && out[cap + i] == 0xA5;
        printf("%zu %llu %d\n", r, h, guard ? 1 : 0);
    }
    return 0;
}
#endif
