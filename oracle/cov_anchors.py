"""Print the line numbers of the source anchors that the quantiser tests must reach (oracle/Makefile writes them to
_ref/cov/anchors.txt).  An anchor is found by its text: the n-th line containing `text` after the first line containing
`after`, so the numbers follow the source they were taken from.  Output: one "name file line" row per anchor.

Build-time tool: the tests read anchors.txt, never the reference sources."""
import os
import sys

# name, after, text, occurrence (1 = first) -- all in SKP_Silk_NSQ_del_dec.c
ANCHORS = [
    # Agora_Silk_RDCx1: the three regions of the two-candidate search (r < -1.5, r > 0.5, in between), each by a
    # rate-distortion line of its own (the regions' first statements are dead stores that carry no count at -O2)
    ("rdcx1_low", "void Agora_Silk_RDCx1(", "rd1_Q10 = SKP_RSHIFT( SKP_SMLABB( SKP_MUL( -SKP_ADD32( q1_Q10", 1),
    ("rdcx1_high", "void Agora_Silk_RDCx1(", "rd1_Q10 = SKP_RSHIFT( SKP_SMLABB( SKP_MUL( SKP_ADD32( q1_Q10", 1),
    ("rdcx1_mid", "void Agora_Silk_RDCx1(", "rd2_Q10 = SKP_RSHIFT( SKP_SMLABB( SKP_MUL( SKP_ADD32( q2_Q10", 2),
    # Agora_Silk_JudgeWinner: a state whose random generator left the winner's, once per sample, once per replacement pass
    ("randsync", "Agora_Silk_JudgeWinner(", "RandSyncCtl++;", 1),
    ("judge_sample", "Agora_Silk_JudgeWinner(", "Winner_rand_state = psDelDec[ Winner_ind ].RandState[ last_smple_idx ];", 1),
    ("judge_pass", "Agora_Silk_JudgeWinner(", "RDmax_Q10  = psSampleState[ 0 ][ 0 ].RD_Q10;", 1),
    # Agora_Silk_DelDec_Rewhitening: the reset of the decisions at sub-frame 2 (interpolated NLSFs only), the rewhitening
    ("reset_k2", "SKP_int32 Agora_Silk_DelDec_Rewhitening(", "RDmin_Q10 = psDelDec[ 0 ].RD_Q10;", 1),
    ("rewhite", "SKP_int32 Agora_Silk_DelDec_Rewhitening(", "start_idx = psEncC->frame_length - lag", 1),
    # SKP_Silk_nsq_del_dec_scale_states: LTP down-scaling of the first rewhitening, rescaling for a new gain
    ("ltp_scale", "void SKP_Silk_nsq_del_dec_scale_states(", "inv_gain_Q32 = SKP_LSHIFT( SKP_SMULWB( inv_gain_Q32, LTP_scale_Q14 ), 2 );", 1),
    ("gain_adj", "void SKP_Silk_nsq_del_dec_scale_states(", "gain_adj_Q16 = SKP_DIV32_varQ( inv_gain_Q16, NSQ->prev_inv_gain_Q16, 16 );", 1),
]


def find(lines, after, text, occurrence):
    start = next(i for i, l in enumerate(lines) if after in l)
    hits = [i for i in range(start, len(lines)) if text in lines[i]]
    return hits[occurrence - 1] + 1


def main(path):
    with open(path, encoding="latin-1") as f:
        lines = f.read().split("\n")
    for name, after, text, occ in ANCHORS:
        print(name, os.path.basename(path), find(lines, after, text, occ))


if __name__ == "__main__":
    main(sys.argv[1])
