/* oracle/record_check.h — the record contract of edge264_b200/csrc/records.h as a check (test infrastructure only). */
#ifndef E264_RECORD_CHECK_H
#define E264_RECORD_CHECK_H
#include "../edge264_b200/csrc/records.h"

/* 0 when the picture keeps the contract; otherwise 1, with the first violation and its macroblock written to why */
int e264_check_records(const E264PicDesc *pd, const E264MbRec *recs, const int16_t *coefs, const E264SliceRec *slices,
                       const uint32_t *intra_list, int n_slots, char *why, int why_len);
/* int16 levels a record owns in the coefficient pool (192 for I_PCM) */
int e264_rec_coef_count(const E264MbRec *r);
#endif
