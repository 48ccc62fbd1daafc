/* lz2_props.h -- TEST INFRASTRUCTURE ONLY.  Forced include (gcc -include) that compiles the oracle for one setting of the LZMA2
 * encoder's literal / position context bits: -DB2ZO_LC=<lc> -DB2ZO_LP=<lp> -DB2ZO_PB=<pb>.
 *
 * The sequential statements (lzma2_enc_oracle.c: stage R; lzma2_opt_oracle.c: stage P through csrc/b2z_lzma_model.h) are written
 * against the compile-time context bits B2Z_LZ2_LC / LP / PB and B2Z_LZ2_PROPS.  Re-binding those macros here, before any of them
 * is expanded, gives a statement of the encoder at that setting, with a model array of the setting's size and the setting's
 * properties byte in the chunk headers -- the bytes the GPU must write when B200Z_P_LZMA2_LC/LP/PB are set to it.  Built by
 * tests/test_oracle_lzma2_props.py (props_oracle) into a temporary directory, one library per setting. */
#ifndef B2ZO_LZ2_PROPS_H
#define B2ZO_LZ2_PROPS_H
#include "b2z_params.h"
#if !defined(B2ZO_LC) || !defined(B2ZO_LP) || !defined(B2ZO_PB)
#error "define B2ZO_LC, B2ZO_LP and B2ZO_PB"
#endif
#if B2ZO_LC + B2ZO_LP > 4 || B2ZO_PB > 4
#error "LZMA2 needs lc + lp <= 4 and pb <= 4"
#endif
#undef B2Z_LZ2_LC
#undef B2Z_LZ2_LP
#undef B2Z_LZ2_PB
#define B2Z_LZ2_LC ((uint32_t)(B2ZO_LC))
#define B2Z_LZ2_LP ((uint32_t)(B2ZO_LP))
#define B2Z_LZ2_PB ((uint32_t)(B2ZO_PB))
#endif
