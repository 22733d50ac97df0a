// consensus_oracle.cpp — test infrastructure: the CPU oracle's own consensus() (oracle/herro_oracle.cpp, included verbatim, not
// restated) on caller-supplied windows, the arguments of hb_consensus_batch.  Built by tests/consensus_oracle.py into tests/_tmp.
#include "../oracle/herro_oracle.cpp"

extern "C" {

// n_reads reads of n_windows[i] windows each, in wid order; per window rows[w] rows of 31 tokens (bases, back to back), n_alns[w],
// and n_sup[w] (pos, ins) pairs (supported) with one row of 5 base logits each (bases_logits).  Writes the segments read after read
// into seqs / seg_len and their count per read into n_segs (0 for None).  Returns 0, or -1 with the read named in ho_last_error
// where the reference would panic.
int ho_consensus_windows(uint32_t n_reads, const uint32_t* n_windows, const uint32_t* rows, const uint8_t* n_alns, const uint8_t* bases,
                         const uint32_t* n_sup, const uint32_t* supported, const float* bases_logits, uint8_t* seqs, uint32_t* seg_len,
                         uint32_t* n_segs) {
    size_t w = 0, row = 0, sup = 0, out = 0, nseg = 0;
    for (uint32_t i = 0; i < n_reads; i++) {
        std::vector<ConsensusWindow> data(n_windows[i]);
        for (uint32_t k = 0; k < n_windows[i]; k++, w++) {
            ConsensusWindow& cw = data[k];
            cw.rid = i;
            cw.wid = (uint16_t)k;
            cw.n_alns = n_alns[w];
            cw.n_total_wins = (uint16_t)n_windows[i];
            cw.bases = Mat(rows[w], TOP_K_SORT + 1, 0);
            std::memcpy(cw.bases.d.data(), bases + row * (TOP_K_SORT + 1), cw.bases.d.size());
            row += rows[w];
            for (uint32_t j = 0; j < n_sup[w]; j++, sup++)
                cw.supported.push_back(SupportedPos{(uint16_t)supported[2 * sup], (uint8_t)supported[2 * sup + 1]});
            cw.has_logits = true;
            cw.info_logits.assign(n_sup[w], 0.0f);
            cw.bases_logits.assign(bases_logits + 5 * (sup - n_sup[w]), bases_logits + 5 * sup);
        }
        std::vector<const ConsensusWindow*> wins;
        for (auto& cw : data) wins.push_back(&cw);
        std::vector<std::vector<uint8_t>> segs;
        try {
            for (auto& cw : data)  // the reference slices n_alns + 1 of the 31 columns
                if (cw.n_alns > TOP_K_SORT) panic("slice end out of bounds: n_alns + 1 columns");
            if (!consensus(wins, segs)) segs.clear();
        } catch (const std::exception& e) {
            g_err = "read " + std::to_string(i) + ": " + e.what();
            return -1;
        }
        n_segs[i] = (uint32_t)segs.size();
        for (auto& s : segs) {
            std::memcpy(seqs + out, s.data(), s.size());
            out += s.size();
            seg_len[nseg++] = (uint32_t)s.size();
        }
    }
    return 0;
}

}  // extern "C"
