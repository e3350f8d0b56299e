// Work decomposition shared by the tensor-core kernels (statistics pre-pass, forward values, backward).
//
// One ITEM = (direction, sample b, line, query tile iq, key block ik):
//   direction : column line (pixels (h, w=line), h = 0..H-1; self entry masked, cc_attention/functions.py:38)
//               or row line (pixels (h=line, w), w = 0..W-1; functions.py:39)
//   query tile: pixels [q0, q0+lq) of the line      key block: pixels [k0, k0+lk) of the line
// Lines up to 112 pixels are one tile; longer lines are cut into nt = ceil(L/112) tiles of equal nominal
// length (queries and keys alike), so the reference's "no size limit" (functions.py:38-47) holds for the tensor-core
// kernels too.  Because every item normalises with the FINAL log-sum-exp of its pixels (left by the statistics
// pre-pass), items are independent: each adds its share of the result onto the output (TMA reduce-add).
//
// Item order (static, round-robin over the persistent CTAs): sample by sample, so that the second touch of a sample's
// tensors (other direction / other tile) finds them in L2; inside a sample
//   segment 0: column items with ik == 0   ("producers": they STORE the output tiles / publish delta; everything another
//   segment 1: column items with ik >= 1    item of the sample may wait for has a LOWER index -> no cyclic waits)
//   segment 2: row items                   ("consumers": they ADD onto what the producers stored)
// decode_item walks the samples one after the other (P(0) C(0) P(1) C(1) ...); decode_item_lagged lets the consumers of a
// sample trail its producers by one block (P(0) P(1) C(0) P(2) C(1) ... C(B-1)): by the time a consumer wants to add onto
// the output, the producers of its sample have long finished, at the price of a larger L2 working set.
// Host + device code: the same functions are unit-tested on the CPU (tests/test_items_host.py via cca_b200_debug_item).
#pragma once

#ifndef __CUDACC__
#define CCA_HD inline
#else
#define CCA_HD __host__ __device__ __forceinline__
#endif

namespace cca {
namespace tc {

constexpr int kMaxTile = 112;   // longest tile (pixels) the kernels handle = largest LK template
constexpr int kMaxNT = 8;       // tiles per line (lines up to 896 pixels)

struct DirGeom {
    int L;    // pixels on a line
    int NL;   // lines per sample
    int nt;   // tiles per line (query tiles == key blocks)
    int tl;   // nominal tile length = ceil(L / nt); the last tile may be shorter
};

struct ItemSpace {
    int B, H, W;
    DirGeom col, row;    // col: L = H, NL = W      row: L = W, NL = H
    int seg0, seg1, seg2;  // items per sample in the three segments
    int per_sample, total;
    int nparts;          // partial log-sum-exp planes the statistics pass leaves per pixel: row.nt + col.nt
};

struct Item {
    int col;             // 1: column line, 0: row line
    int b, line, iq, ik;
    int q0, lq, k0, lk;
    int j;               // index of the item inside its sample (0 .. per_sample-1)
};

CCA_HD int tiles_for(int L) { return (L + kMaxTile - 1) / kMaxTile; }

CCA_HD DirGeom make_dir(int L, int NL)
{
    DirGeom g;
    g.L = L; g.NL = NL;
    g.nt = tiles_for(L);
    g.tl = (L + g.nt - 1) / g.nt;
    return g;
}

CCA_HD ItemSpace make_space(int B, int H, int W)
{
    ItemSpace s;
    s.B = B; s.H = H; s.W = W;
    s.col = make_dir(H, W);
    s.row = make_dir(W, H);
    s.seg0 = s.col.NL * s.col.nt;
    s.seg1 = s.col.NL * s.col.nt * (s.col.nt - 1);
    s.seg2 = s.row.NL * s.row.nt * s.row.nt;
    s.per_sample = s.seg0 + s.seg1 + s.seg2;
    s.total = B * s.per_sample;
    s.nparts = s.row.nt + s.col.nt;
    return s;
}

// longest tile of either direction (selects the LK template: 80 or 112)
CCA_HD int max_tile(const ItemSpace &s) { return s.col.tl > s.row.tl ? s.col.tl : s.row.tl; }

CCA_HD Item decode_item(const ItemSpace &s, int idx)
{
    Item it;
    it.b = idx / s.per_sample;
    int j = idx - it.b * s.per_sample;
    it.j = j;
    const DirGeom *g;
    if (j < s.seg0) {                       // column, ik == 0
        it.col = 1; g = &s.col;
        it.line = j / g->nt; it.iq = j - it.line * g->nt; it.ik = 0;
    } else if (j < s.seg0 + s.seg1) {       // column, ik >= 1
        it.col = 1; g = &s.col;
        j -= s.seg0;
        const int per = g->nt - 1;
        const int li = j / per;             // line * nt + iq
        it.ik = 1 + (j - li * per);
        it.line = li / g->nt; it.iq = li - it.line * g->nt;
    } else {                                // row
        it.col = 0; g = &s.row;
        j -= s.seg0 + s.seg1;
        const int li = j / g->nt;
        it.ik = j - li * g->nt;
        it.line = li / g->nt; it.iq = li - it.line * g->nt;
    }
    it.q0 = it.iq * g->tl; it.k0 = it.ik * g->tl;
    it.lq = g->L - it.q0 < g->tl ? g->L - it.q0 : g->tl;
    it.lk = g->L - it.k0 < g->tl ? g->L - it.k0 : g->tl;
    return it;
}

// item j (0 .. per_sample-1) of sample b
CCA_HD Item decode_item_in_sample(const ItemSpace &s, int b, int j) { return decode_item(s, b * s.per_sample + j); }

// P(0) | P(1) C(0) | P(2) C(1) | ... | P(B-1) C(B-2) | C(B-1)      P(b) = segment 0 of sample b, C(b) = segments 1, 2
CCA_HD Item decode_item_lagged(const ItemSpace &s, int idx)
{
    const int np = s.seg0, nc = s.per_sample - s.seg0;
    if (idx < np) return decode_item_in_sample(s, 0, idx);
    const int x = idx - np;
    const int grp = x / s.per_sample, rem = x - grp * s.per_sample;
    if (grp < s.B - 1) {
        if (rem < np) return decode_item_in_sample(s, grp + 1, rem);
        return decode_item_in_sample(s, grp, np + (rem - np));
    }
    (void)nc;
    return decode_item_in_sample(s, s.B - 1, np + rem);
}
CCA_HD Item decode_item_order(const ItemSpace &s, int idx, int lag) { return lag ? decode_item_lagged(s, idx) : decode_item(s, idx); }
// segment-0 items ("producers") of a sample
CCA_HD bool is_producer(const Item &it) { return it.col && it.ik == 0; }

// pixel index (b, h, w) -> flat [B,H,W] of query row r of an item
CCA_HD long item_pixel(const ItemSpace &s, const Item &it, int r)
{
    return it.col ? ((long)it.b * s.H + (it.q0 + r)) * s.W + it.line : ((long)it.b * s.H + it.line) * s.W + (it.q0 + r);
}
// plane of the partial log-sum-exp this (direction, key block) writes / all items read: rows first, then columns
CCA_HD int part_index(const ItemSpace &s, const Item &it) { return it.col ? s.row.nt + it.ik : it.ik; }
// plane of the (direction, query tile) partial dK / dV of the deterministic backward (cca_tc_bwd.cuh, planes mode)
CCA_HD int qtile_part_index(const ItemSpace &s, const Item &it) { return it.col ? s.row.nt + it.iq : it.iq; }

// Zero-ahead: the items of sample b clear the output of sample b + ahead before anybody adds onto it.  Item j of a sample
// owns bytes [j*share, min(bytes, (j+1)*share)) of that sample's slice of each output tensor.
CCA_HD long zero_share_bytes(long sample_bytes, int per_sample)
{
    const long s = (sample_bytes + per_sample - 1) / per_sample;
    return (s + 127) / 128 * 128;
}

}  // namespace tc
}  // namespace cca
