// dfa_tables.cpp -- see dfa_tables.hpp.
#include "dfa_tables.hpp"

#include <algorithm>
#include <numeric>

namespace pire_b200 {

std::vector<uint32_t> StaticHotOrder(const Dfa& dfa)
{
    std::vector<uint32_t> order;
    std::vector<uint8_t> seen(dfa.states, 0);
    order.reserve(dfa.states);
    auto push = [&](uint32_t s) {
        if (!seen[s]) {
            seen[s] = 1;
            order.push_back(s);
        }
    };
    // The state every string is in after Begin() comes first, then Initialize().
    push(dfa.Next(dfa.initial, kBeginMark));
    push(dfa.initial);
    for (size_t head = 0; head < order.size(); ++head) {
        uint32_t s = order[head];
        for (uint32_t b = 0; b < 256; ++b)
            push(dfa.Next(s, b));
    }
    for (uint32_t s = 0; s < dfa.states; ++s)   // unreachable by bytes (only by marks)
        push(s);
    return order;
}

std::vector<uint32_t> HotOrderFromCounts(const Dfa& dfa, const std::vector<uint64_t>& visits)
{
    std::vector<uint32_t> fallback = StaticHotOrder(dfa);
    std::vector<uint32_t> rank(dfa.states);
    for (uint32_t i = 0; i < dfa.states; ++i)
        rank[fallback[i]] = i;
    std::vector<uint32_t> order(dfa.states);
    std::iota(order.begin(), order.end(), 0u);
    std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) {
        uint64_t va = a < visits.size() ? visits[a] : 0, vb = b < visits.size() ? visits[b] : 0;
        if (va != vb)
            return va > vb;
        return rank[a] < rank[b];
    });
    return order;
}

void BuildScanTables(const Dfa& dfa, const std::vector<uint32_t>& hot_order, uint32_t max_hot, ScanTables* out)
{
    ScanTables& t = *out;
    t = ScanTables();
    t.states = dfa.states;
    t.letters = dfa.letters;
    t.hot = std::min<uint32_t>(std::min<uint32_t>(kMaxHot, max_hot), dfa.states);
    if (t.hot == 0)
        t.hot = 1;
    const uint32_t H = t.hot;

    // Renumber: hot states first (in hot_order), the rest in their old order.
    t.new_of_old.assign(dfa.states, UINT32_MAX);
    t.old_of_new.clear();
    t.old_of_new.reserve(dfa.states);
    for (uint32_t s : hot_order) {
        if (t.old_of_new.size() == H)
            break;
        if (s < dfa.states && t.new_of_old[s] == UINT32_MAX) {
            t.new_of_old[s] = 0;
            t.old_of_new.push_back(s);
        }
    }
    // Final hot states take the highest hot ids (order otherwise kept): the counting and prefix kernels
    // then learn "did this chunk enter a final state or leave the hot rows" from the maximum id seen.
    std::stable_partition(t.old_of_new.begin(), t.old_of_new.end(), [&](uint32_t s) { return !dfa.Final(s); });
    t.first_final_hot = (uint32_t) t.old_of_new.size();
    for (uint32_t k = 0; k < t.old_of_new.size(); ++k) {
        t.new_of_old[t.old_of_new[k]] = k;
        if (dfa.Final(t.old_of_new[k]) && t.first_final_hot == t.old_of_new.size())
            t.first_final_hot = k;
    }
    for (uint32_t s = 0; s < dfa.states; ++s)
        if (t.new_of_old[s] == UINT32_MAX) {
            t.new_of_old[s] = (uint32_t) t.old_of_new.size();
            t.old_of_new.push_back(s);
        }

    t.cls.resize(256);
    for (uint32_t b = 0; b < 256; ++b)
        t.cls[b] = dfa.class_of[b];

    // Complete table in the new numbering.
    t.wide = dfa.states > 65536;
    const size_t cells = (size_t) dfa.states * dfa.letters;
    if (t.wide)
        t.full32.resize(cells);
    else
        t.full16.resize(cells);
    for (uint32_t ns = 0; ns < dfa.states; ++ns) {
        const uint32_t* row = &dfa.next[(size_t) t.old_of_new[ns] * dfa.letters];
        for (uint32_t c = 0; c < dfa.letters; ++c) {
            uint32_t to = t.new_of_old[row[c]];
            if (t.wide)
                t.full32[(size_t) ns * dfa.letters + c] = to;
            else
                t.full16[(size_t) ns * dfa.letters + c] = (uint16_t) to;
        }
    }

    // Fused hot rows.
    t.hot8.assign(HotTableBytes(H), (uint8_t) H);
    t.noexit.assign(H + 1, 0);
    for (uint32_t h = 0; h < H; ++h) {
        const uint32_t* row = &dfa.next[(size_t) t.old_of_new[h] * dfa.letters];
        bool stays = true;
        for (uint32_t b = 0; b < 256; ++b) {
            uint32_t to = t.new_of_old[row[dfa.class_of[b]]];
            t.hot8[(size_t) h * kHotStride + b] = (uint8_t) (to < H ? to : H);
            stays = stays && to == h;
        }
        t.noexit[h] = stays ? 1 : 0;    // same predicate as BuildShortcuts' NoExit, multi.h:477-514
    }

    // 32-slot filter of the kPred variant: slot = byte & 31.
    t.exit_bitmap0 = 0;
    for (uint32_t b = 0; b < 256; ++b)
        if (t.hot8[b] != 0)
            t.exit_bitmap0 |= 1u << (b & 31);

    // Look-ahead filter of the LOOK variant.  F1 = bytes that leave id 0; F = F1 plus every byte on which a state
    // entered from id 0 goes anywhere but back to id 0.  If byte k+1 is outside F, then whatever byte k did to a lane
    // resting in id 0, the lane is back in id 0 after byte k+1: both table reads can be skipped.
    t.look_ok = true;
    {
        bool in_f[256];
        for (uint32_t b = 0; b < 256; ++b)
            in_f[b] = t.hot8[b] != 0;
        for (uint32_t b = 0; b < 256; ++b) {
            const uint32_t g1 = t.hot8[b];
            if (g1 == 0)
                continue;
            if (g1 >= H) {
                t.look_ok = false;
                break;
            }
            for (uint32_t c = 0; c < 256; ++c)
                if (t.hot8[(size_t) g1 * kHotStride + c] != 0)
                    in_f[c] = true;
        }
        t.look_bitmap = 0;
        t.look_bitmap64 = 0;
        for (uint32_t b = 0; b < 256; ++b)
            if (in_f[b]) {
                t.look_bitmap |= 1u << (b & 31);
                t.look_bitmap64 |= 1ull << (b & 63);
            }
        if (!t.look_ok) {
            t.look_bitmap = ~0u;
            t.look_bitmap64 = ~0ull;
        }
    }

    // Lane-private rows: as many of the hottest states as fit, rounded to whole quads,
    // the last id being the sink.
    {
        uint32_t real = std::min<uint32_t>(H, kMaxPrivRows - 1);
        uint32_t rows = (real + 1 + 3) / 4 * 4;
        real = std::min<uint32_t>(H, rows - 1);
        const uint32_t sink = rows - 1;
        t.priv_rows = rows;
        t.priv_packed.assign((size_t) (rows / 4) * 128, 0);
        for (uint32_t r = 0; r < rows; ++r)
            for (uint32_t b = 0; b < 128; ++b) {
                uint32_t to = sink;
                if (r < real) {
                    uint32_t h = t.hot8[(size_t) r * kHotStride + b];
                    if (h < real)
                        to = h;
                }
                t.priv_packed[(size_t) (r / 4) * 128 + b] |= to << (8 * (r % 4));
            }
    }

    {
        const uint32_t Hs = std::min<uint32_t>(H, kPrivHotRows);
        t.hot_small = Hs;
        t.hot8_small.assign(HotTableBytes(Hs), (uint8_t) Hs);
        for (uint32_t h = 0; h < Hs; ++h)
            for (uint32_t b = 0; b < 256; ++b) {
                uint32_t to = t.hot8[(size_t) h * kHotStride + b];
                t.hot8_small[(size_t) h * kHotStride + b] = (uint8_t) (to < Hs ? to : Hs);
            }
    }

    // What a string that stops in state s reports.
    for (int with_end = 0; with_end < 2; ++with_end) {
        t.fin[with_end].resize(dfa.states);
        for (uint32_t ns = 0; ns < dfa.states; ++ns) {
            uint32_t os = t.old_of_new[ns];
            uint32_t last = with_end ? dfa.Next(os, kEndMark) : os;      // RunHelper::End(), run.h:376
            FinEntry f;
            f.result = last | (dfa.Final(last) ? 0x80000000u : 0u);      // operator bool, run.h:380-381
            f.mask = 0;
            for (uint32_t k = dfa.acc_begin[last]; k < dfa.acc_begin[last + 1]; ++k)
                if (dfa.acc_ids[k] < 32)
                    f.mask |= 1u << dfa.acc_ids[k];                      // AcceptedRegexps, multi.h:149-158
            t.fin[with_end][ns] = f;
        }
    }

    t.flags_new.resize(dfa.states);
    for (uint32_t ns = 0; ns < dfa.states; ++ns)
        t.flags_new[ns] = dfa.flags[t.old_of_new[ns]];
    t.end_class = dfa.class_of[kEndMark];
    t.begin_class = dfa.class_of[kBeginMark];
    t.initial = t.new_of_old[dfa.initial];
    t.acc_begin_new.assign((size_t) dfa.states + 1, 0);
    t.acc_ids_new.clear();
    for (uint32_t ns = 0; ns < dfa.states; ++ns) {
        t.acc_begin_new[ns] = (uint32_t) t.acc_ids_new.size();
        const uint32_t os = t.old_of_new[ns];
        if (!dfa.Final(os))                      // TakeAction only looks at the list of a final state
            continue;
        for (uint32_t k = dfa.acc_begin[os]; k < dfa.acc_begin[os + 1]; ++k)
            if (dfa.acc_ids[k] < std::max<uint32_t>(1, dfa.regexps))     // a counter exists for it
                t.acc_ids_new.push_back(dfa.acc_ids[k]);
    }
    t.acc_begin_new[dfa.states] = (uint32_t) t.acc_ids_new.size();

    const uint32_t regs = std::max<uint32_t>(1, dfa.regexps);
    t.count_words = regs <= 16 ? (regs + 7) / 8 : 0;
    t.weights.assign((size_t) dfa.states * t.count_words, 0);
    for (uint32_t ns = 0; ns < dfa.states && t.count_words; ++ns) {
        uint32_t times[16] = {0};
        for (uint32_t k = t.acc_begin_new[ns]; k < t.acc_begin_new[ns + 1]; ++k)
            ++times[t.acc_ids_new[k]];
        for (uint32_t r = 0; r < regs; ++r) {
            if (times[r] > 15) {
                t.count_words = 0;
                t.weights.clear();
                break;
            }
            t.weights[(size_t) ns * t.count_words + r / 8] |= (uint64_t) times[r] << (8 * (r % 8));
        }
    }

    // The ids still acceptable from each state: a fixpoint over the transitions, propagated backwards from the final
    // states' accept lists with a worklist over the predecessors.
    t.live_words = (regs + 31) / 32;
    t.live.assign((size_t) dfa.states * t.live_words, 0);
    {
        const uint32_t W = t.live_words;
        std::vector<uint32_t> pred_begin((size_t) dfa.states + 1, 0), preds((size_t) dfa.states * dfa.letters);
        for (uint32_t ns = 0; ns < dfa.states; ++ns)
            for (uint32_t c = 0; c < dfa.letters; ++c)
                ++pred_begin[(t.wide ? t.full32[(size_t) ns * dfa.letters + c] : t.full16[(size_t) ns * dfa.letters + c]) + 1];
        for (uint32_t ns = 0; ns < dfa.states; ++ns)
            pred_begin[ns + 1] += pred_begin[ns];
        std::vector<uint32_t> fill(pred_begin.begin(), pred_begin.end() - 1);
        for (uint32_t ns = 0; ns < dfa.states; ++ns)
            for (uint32_t c = 0; c < dfa.letters; ++c)
                preds[fill[t.wide ? t.full32[(size_t) ns * dfa.letters + c] : t.full16[(size_t) ns * dfa.letters + c]]++] = ns;
        std::vector<uint32_t> work;
        for (uint32_t ns = 0; ns < dfa.states; ++ns) {
            for (uint32_t k = t.acc_begin_new[ns]; k < t.acc_begin_new[ns + 1]; ++k)
                t.live[(size_t) ns * W + t.acc_ids_new[k] / 32] |= 1u << (t.acc_ids_new[k] % 32);
            work.push_back(ns);
        }
        while (!work.empty()) {
            const uint32_t s = work.back();
            work.pop_back();
            const uint32_t* from = &t.live[(size_t) s * W];
            for (uint32_t k = pred_begin[s]; k < pred_begin[s + 1]; ++k) {
                uint32_t* to = &t.live[(size_t) preds[k] * W];
                bool grew = false;
                for (uint32_t w = 0; w < W; ++w)
                    if (from[w] & ~to[w]) {
                        to[w] |= from[w];
                        grew = true;
                    }
                if (grew)
                    work.push_back(preds[k]);
            }
        }
    }

    t.start[0] = t.new_of_old[dfa.initial];                              // Initialize(), multi.h:161
    t.start[1] = t.new_of_old[dfa.Next(dfa.initial, kBeginMark)];        // Begin(), run.h:375
}

} // namespace pire_b200
