/* parse_counts.c — dynamic counts of the fast greedy parse (K1b, zb_parse_kernel) on one input, CPU only.
 *
 *   make -C oracle oracle && cc -O2 -o /tmp/parse_counts tools/parse_counts.c -Loracle -lzb_oracle -Wl,-rpath,$PWD/oracle
 *   oracle/_ref/datagen -g256MB -P50 > /tmp/p50 && /tmp/parse_counts /tmp/p50 1
 *
 * The input is compressed as one frame.  The candidates come from the oracle's walk (zbo_walkChunk, bit-exact with
 * K1a); the parse below makes the same steps, lanes and winners as parse_fast_segment in oracle/zb_match.c (the rule
 * both the kernel and the oracle follow) and counts, per segment, what the kernel does on its way:
 *   steps             probe steps (32 lanes each);
 *   hits by type      repcode 2 (lane 0 at the anchor), repcode 1, table;
 *   tried             table lanes the kernel tries: a lane whose repcodes failed and whose candidate is non-zero and, if
 *                     below 0xFFFF, does not reach in front of the history — the far ones are tried whatever their reach;
 *   tag false         tried lanes whose first 4 bytes differ (the walk only checks an 11-bit tag);
 *   far               tried lanes with a distance >= 0xFFFF (the kernel fetches the 32-bit distance for each), far winners;
 *   fwd rounds        256-byte rounds of forward compares per match (floor(counted / 256) + 1, counted from the probe for
 *                     a table hit, from probe + 4 for a repcode hit);
 *   back rounds       32-byte rounds of backward catch-up per match (floor(back / 32) + 1);
 *   back > 4          matches whose catch-up exceeds 4 bytes (the in-lane repcode-1 catch-up of the kernel before stopped there);
 *   catch-up split    matches whose catch-up lane 31's 8-byte window answers (fewer than 8 bytes) and those that go on to
 *                     the cooperative 32-byte rounds (8 or more); the forward rounds past the first window (31 lanes,
 *                     248 bytes, then 256 per round);
 *   pairs             iterations of the current kernel, which probes two steps per iteration (a pair of positions per
 *                     lane); its winners in the first half (the step at ip) and in the second (the step after it), and
 *                     those found in a later iteration than the first after the anchor; tries per iteration.
 * From these it prints the dependent memory round trips per segment of four kernels: two per step; one per step with a
 * hit's first rounds waiting twice; one per step with a hit's windows all out before the first is compared; and the
 * current one, one per iteration of two steps (DESIGN.md section 2, K1b).  It also prints the issue floor of config 2 of
 * the last two kernels from their SASS instruction counts. */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "../oracle/zb_oracle.h"

/* warp instructions of zb_parse_kernel<false> per path, counted in `cuobjdump -sass` of the sm_90a build (DESIGN.md
 * section 10): one step of one position per lane without a hit and with a table hit (through the store of the
 * sequence), and the same for one iteration of the pair kernel (two steps, a pair of positions per lane) */
#define SASS_STEP_MISS 84
#define SASS_STEP_HIT 216
#define SASS_PAIR_MISS 88
#define SASS_PAIR_HIT 239

static u32 rd32(const u8* p) { u32 v; memcpy(&v, p, 4); return v; }
static size_t count_eq(const u8* a, const u8* b, const u8* end) { const u8* s = a; while (a < end && *a == *b) { a++; b++; } return (size_t)(a - s); }

typedef struct {
    double segs, steps, matches, h3, h2, h1, tried, tagFalse, farTried, farLost, farWon, fwdRounds, backRounds, back4,
           fwdExtra, backExtra, backRoundsTable, rep1Coop, backInWin, backCoop, fwdExtraWin, backExtraWin,
           iters, winFirstHalf, winSecondHalf, winLater;
} counts;

/* two steps of the rule per iteration of the pair kernel: a match found after j steps without a hit is found in iteration
 * j / 2 after the anchor, in its first half when j is even; s steps without a hit at a segment's end take (s + 1) / 2 */
static void pair_iters(counts* c, double j, int hit)
{
    if (!hit) { c->iters += (double)(((size_t)j + 1) / 2); return; }
    c->iters += (double)((size_t)j / 2 + 1);
    if ((size_t)j % 2 == 0) c->winFirstHalf++; else c->winSecondHalf++;
    if (j >= 2) c->winLater++;
}

static void parse_segment(const zbo_plan* plan, const u8* frame, const u32* dist, size_t bs, size_t be, size_t ss, size_t se,
                          size_t lowLimit, counts* c)
{
    size_t ip = ss, anchor = ss, searchStart = ss;
    u32 rep1 = 0, rep2 = 0;
    double misses = 0;                                   /* steps without a hit since the anchor */
    c->segs++;
    while (ip < se && ip + 8 <= be) {
        u32 const step = plan->stepSize + (u32)((ip - searchStart) >> 7);
        int winner = -1, wtype = 0, l;
        size_t probe = 0; u32 offset = 0;
        c->steps++;
        for (l = 0; l < (int)ZB_WARP && winner < 0; l++) {
            size_t const p = ip + (size_t)(l >> 1) * step + (size_t)(l & 1);
            u32 cur, d;
            if (p >= se || p + 8 > be) break;
            cur = rd32(frame + p);
            d = dist[p - bs];
            if (l == 0 && ip == anchor && rep2 && rd32(frame + p - rep2) == cur) { winner = l; wtype = 3; probe = p; offset = rep2; }
            else if (rep1 && p >= lowLimit + rep1 && rd32(frame + p - rep1) == cur) { winner = l; wtype = 2; probe = p; offset = rep1; }
            else if (d && (d >= 0xFFFFu || p >= lowLimit + d)) {
                c->tried++;
                if (d >= 0xFFFFu) c->farTried++;
                if (p < lowLimit + d) { c->farLost++; continue; }
                if (rd32(frame + p - d) != cur) { c->tagFalse++; continue; }
                winner = l; wtype = 1; probe = p; offset = d;
                if (d >= 0xFFFFu) c->farWon++;
            }
        }
        if (winner < 0) { misses++; ip += (size_t)(ZB_WARP / 2) * step; continue; }
        pair_iters(c, misses, 1);
        misses = 0;
        {   size_t ms = probe, mm = probe - offset, mlen, fwd, back;
            if (wtype != 3)
                while (ms > anchor && mm > lowLimit && frame[ms - 1] == frame[mm - 1]) { ms--; mm--; }
            fwd = count_eq(frame + probe + 4, frame + probe - offset + 4, frame + be);
            mlen = (probe - ms) + 4 + fwd;
            back = probe - ms;
            c->matches++;
            if (wtype == 3) c->h3++; else if (wtype == 2) c->h2++; else c->h1++;
            {   size_t const counted = (wtype == 1) ? fwd + 4 : fwd;
                c->fwdRounds += (double)(counted / 256 + 1);
                c->fwdExtra += (double)(counted / 256);
            }
            c->backRounds += (double)(back / 32 + 1);
            c->backExtra += (double)(back / 32);
            if (wtype == 1) c->backRoundsTable += (double)(back / 32 + 1);
            if (back > 4) { c->back4++; if (wtype == 2) c->rep1Coop += (double)((back - 4) / 32 + 1); }
            if (back < 8) c->backInWin++;
            else { c->backCoop++; c->backExtraWin += (double)((back - 8) / 32 + 1); }
            {   size_t const counted = (wtype == 1) ? fwd + 4 : fwd;
                if (counted >= 248) c->fwdExtraWin += (double)((counted - 248) / 256 + 1);
            }
            if (wtype == 3) { u32 const t = rep2; rep2 = rep1; rep1 = t; }
            else if (wtype == 1) { rep2 = rep1; rep1 = offset; }
            ip = ms + mlen; anchor = ip; searchStart = ip;
        }
    }
    pair_iters(c, misses, 0);
}

int main(int argc, char** argv)
{
    FILE* f;
    u8* src;
    size_t n, bs;
    int level = argc > 2 ? atoi(argv[2]) : 1;
    zbo_cparams cp;
    zbo_plan plan;
    zbo_chunkCand cc;
    counts c;
    if (argc < 2) { fprintf(stderr, "usage: %s <input> [level]\n", argv[0]); return 2; }
    f = fopen(argv[1], "rb");
    if (!f) { perror(argv[1]); return 1; }
    fseek(f, 0, SEEK_END); n = (size_t)ftell(f); fseek(f, 0, SEEK_SET);
    src = (u8*)malloc(n + 16);
    if (fread(src, 1, n, f) != n) { fprintf(stderr, "short read\n"); return 1; }
    fclose(f);
    cp = zbo_getCParams(level, n, 0);
    if (cp.strategy != 1) { fprintf(stderr, "level %d is not the fast strategy\n", level); return 2; }
    zbo_makePlan(&plan, &cp);
    memset(&c, 0, sizeof c);
    memset(&cc, 0, sizeof cc);
    {   size_t const chunkBytes = (size_t)plan.chunkBlocks * ZB_BLOCK_MAX;
        for (bs = 0; bs < n; bs += ZB_BLOCK_MAX) {
            size_t const be = bs + ZB_BLOCK_MAX < n ? bs + ZB_BLOCK_MAX : n, W = (size_t)1 << plan.windowLog;
            size_t lowLimit, ss;
            if (bs % chunkBytes == 0) {
                size_t const ce = bs + chunkBytes < n ? bs + chunkBytes : n;
                zbo_freeChunk(&cc);
                zbo_walkChunk(&plan, src, n, bs, ce, &cc);
            }
            if (be - bs < 7) continue;                           /* raw block, no parse */
            lowLimit = cc.low;                                   /* oracle/zb_match.c block_low */
            if (be > W && be - W > lowLimit) lowLimit = be - W;
            for (ss = bs; ss < be; ss += ZB_PARSE_SEG)
                parse_segment(&plan, src, cc.dS + (bs - cc.start), bs, be, ss, ss + ZB_PARSE_SEG < be ? ss + ZB_PARSE_SEG : be, lowLimit, &c);
        }
        zbo_freeChunk(&cc);
    }
    {   double const S = c.segs, M = c.matches;
        /* before: 2 round trips per step (the dist row, then the windows and the far distance); per match the forward
         * rounds and the backward rounds of a table hit or of a repcode-1 hit with more than 4 bytes of catch-up, plus one
         * for the repcode-1 in-lane catch-up's window; one forward round per tried false positive.
         * waiting twice: 1 per step, 1 per far lane tried; per match and per tried false positive the first forward and
         * backward rounds, which went out together but waited twice in the sm_90a SASS (the compare of the current window
         * was scheduled before the loads of the candidate window and of the catch-up bytes), then the extra rounds of each;
         * once: the same, but a hit's two windows per lane (lane 31's holding the catch-up) wait once, and the extra rounds
         * start past 248 bytes forward and 8 bytes backward;
         * pairs: the same per iteration of two steps as per step before */
        double const rtOld = 2 * c.steps + c.fwdRounds + c.backRoundsTable + c.h2 + c.rep1Coop + c.tagFalse;
        double const rtTwice = c.steps + c.farTried + 2 * (M + c.tagFalse) + c.fwdExtra + c.backExtra;
        double const rtOnce = c.steps + c.farTried + (M + c.tagFalse) + c.fwdExtraWin + c.backExtraWin;
        double const rtPairs = c.iters + c.farTried + (M + c.tagFalse) + c.fwdExtraWin + c.backExtraWin;
        /* issue floor of config 2: 1 GiB in 16 KiB segments on the 132 SMs of an H100, 4 warp instructions per cycle per SM
         * at 1980 MHz, the instructions per segment from the SASS counts above (tag false positives and far fetches left
         * out of both) */
        double const floorK = 65536.0 / (132.0 * 4.0 * 1980e6) * 1e3;
        double const instStep = (c.steps - M) * SASS_STEP_MISS + M * SASS_STEP_HIT;
        double const instPair = (c.iters - M) * SASS_PAIR_MISS + M * SASS_PAIR_HIT;
        printf("{\"input_bytes\": %zu, \"level\": %d, \"segments\": %.0f, \"per_segment\": {\"steps\": %.2f, \"matches\": %.2f, "
               "\"rep2\": %.2f, \"rep1\": %.2f, \"table\": %.2f, \"tried\": %.2f, \"tag_false\": %.3f, \"far_tried\": %.3f, "
               "\"far_out_of_reach\": %.3f, \"far_won\": %.3f, \"back_gt4\": %.2f, \"fwd_rounds\": %.2f, \"back_rounds\": %.2f, "
               "\"catchup_in_window\": %.2f, \"catchup_cooperative\": %.2f, \"fwd_past_window\": %.2f}, "
               "\"per_match\": {\"steps\": %.3f, \"fwd_rounds\": %.3f, \"back_rounds\": %.3f}, "
               "\"pairs_per_segment\": {\"iterations\": %.2f, \"win_first_half\": %.2f, \"win_second_half\": %.2f, "
               "\"win_later_iteration\": %.2f, \"tries_per_iteration\": %.3f, \"iterations_per_match\": %.3f}, "
               "\"round_trips_per_segment\": {\"two_per_step\": %.1f, \"hit_waits_twice\": %.1f, \"hit_waits_once\": %.1f, "
               "\"pairs\": %.1f}, "
               "\"issue_floor_ms\": {\"one_step_per_iteration\": %.2f, \"pairs\": %.2f}, \"instructions_per_match\": {\"one_step_per_iteration\": %.1f, "
               "\"pairs\": %.1f}}\n",
               n, level, S, c.steps / S, M / S, c.h3 / S, c.h2 / S, c.h1 / S, c.tried / S, c.tagFalse / S, c.farTried / S,
               c.farLost / S, c.farWon / S, c.back4 / S, c.fwdRounds / S, c.backRounds / S,
               c.backInWin / S, c.backCoop / S, c.fwdExtraWin / S,
               c.steps / M, c.fwdRounds / M, c.backRounds / M,
               c.iters / S, c.winFirstHalf / S, c.winSecondHalf / S, c.winLater / S, (c.tried + c.h2 + c.h3) / c.iters, c.iters / M,
               rtOld / S, rtTwice / S, rtOnce / S, rtPairs / S,
               floorK * instStep / S, floorK * instPair / S, instStep / M, instPair / M);
    }
    free(src);
    return 0;
}
