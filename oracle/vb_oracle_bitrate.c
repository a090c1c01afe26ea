/* vb_oracle_bitrate.c — the CPU oracle of the bitrate manager.  TEST INFRASTRUCTURE ONLY.
 *
 * A plain-C restatement of vorbis_bitrate_init (lib/bitrate.c:28-56) and vorbis_bitrate_addblock (:73-227) on
 * packet lengths alone: the 15 packets of a block are given as bit counts, and the result is the packet kept and its
 * final length in bytes (cut to maxsize, or padded with zero bytes up to minsize).  It is written from the reference's
 * description, not shared with the device code (vorbis_b200/csrc/vb200_bitrate.cuh), so that each checks the other.
 * Built into oracle/libvb_oracle_bitrate.so by oracle/bitrate.py, anywhere gcc exists.
 */
#include <math.h>
#include <string.h>

#include "vorbis_b200.h"

#define NB VB200_PACKETBLOBS

/* bitrate_manager_state's constants, as vorbis_bitrate_init derives them */
typedef struct vbo_bitrate {
  long avg_bitsper, min_bitsper, max_bitsper, short_per_long;
  long desired_fill;
  long reservoir_bits;
  double slew_damp;
  long rate;
  int blocksizes[2];
} vbo_bitrate;

/* the branches of one run, for the tests' coverage: [0] slew-down steps, [1] slew-up steps, [2] min-loop steps,
 * [3] max-loop steps, [4] truncated packets, [5] padded packets */
#define VBO_BR_BRANCHES 6

/* returns 0, or -1 for an un-managed info (reservoir_bits <= 0) */
int vbo_bitrate_derive(const vb200_bitrate_info *bi, long rate, int bs0, int bs1, vbo_bitrate *B){
  const int halfsamples = bs0 >> 1;
  memset(B, 0, sizeof(*B));
  if(bi->reservoir_bits <= 0) return -1;
  B->short_per_long = bs1 / bs0;
  B->avg_bitsper = rint(1. * bi->avg_rate * halfsamples / rate);
  B->min_bitsper = rint(1. * bi->min_rate * halfsamples / rate);
  B->max_bitsper = rint(1. * bi->max_rate * halfsamples / rate);
  B->desired_fill = bi->reservoir_bits * bi->reservoir_bias;
  B->reservoir_bits = bi->reservoir_bits;
  B->slew_damp = bi->slew_damp;
  B->rate = rate;
  B->blocksizes[0] = bs0; B->blocksizes[1] = bs1;
  return 0;
}

void vbo_bitrate_fresh(const vbo_bitrate *B, vb200_bitrate_state *st){
  memset(st, 0, sizeof(*st));
  st->avg_reservoir = st->minmax_reservoir = B->desired_fill;
  st->avgfloat = NB / 2;
}

static long blob_bits(const int *bits, int k){ return (long)((bits[k] + 7) / 8) * 8; }

/* one block: bits[NB] the packets' lengths in bits.  Returns the packet kept; *bytes its final length. */
int vbo_bitrate_addblock(const vbo_bitrate *B, int W, const int *bits, vb200_bitrate_state *st, long *bytes,
                         long *branches){
  const long min_target = W ? B->min_bitsper * B->short_per_long : B->min_bitsper;
  const long max_target = W ? B->max_bitsper * B->short_per_long : B->max_bitsper;
  const long avg_target = W ? B->avg_bitsper * B->short_per_long : B->avg_bitsper;
  const int samples = B->blocksizes[W] >> 1;
  int choice = rint(st->avgfloat);
  long this_bits = blob_bits(bits, choice), natural;

  if(B->avg_bitsper > 0){
    const double slewlimit = 15. / B->slew_damp;
    double slew;
    if(st->avg_reservoir + (this_bits - avg_target) > B->desired_fill){
      while(choice > 0 && this_bits > avg_target && st->avg_reservoir + (this_bits - avg_target) > B->desired_fill){
        choice--; this_bits = blob_bits(bits, choice); branches[0]++;
      }
    }else if(st->avg_reservoir + (this_bits - avg_target) < B->desired_fill){
      while(choice + 1 < NB && this_bits < avg_target && st->avg_reservoir + (this_bits - avg_target) < B->desired_fill){
        choice++; this_bits = blob_bits(bits, choice); branches[1]++;
      }
    }
    slew = rint(choice - st->avgfloat) / samples * B->rate;
    if(slew < -slewlimit) slew = -slewlimit;
    if(slew > slewlimit) slew = slewlimit;
    st->avgfloat += slew / B->rate * samples;
    choice = rint(st->avgfloat);
    this_bits = blob_bits(bits, choice);
  }
  if(B->min_bitsper > 0 && this_bits < min_target){
    while(st->minmax_reservoir - (min_target - this_bits) < 0){
      branches[2]++;
      if(++choice >= NB) break;
      this_bits = blob_bits(bits, choice);
    }
  }
  if(B->max_bitsper > 0 && this_bits > max_target){
    while(st->minmax_reservoir + (this_bits - max_target) > B->reservoir_bits){
      branches[3]++;
      if(--choice < 0) break;
      this_bits = blob_bits(bits, choice);
    }
  }
  if(choice < 0){
    const long maxsize = (max_target + (B->reservoir_bits - st->minmax_reservoir)) / 8;
    choice = 0;
    natural = (bits[0] + 7) / 8;
    *bytes = natural > maxsize ? (maxsize > 0 ? maxsize : 0) : natural;
  }else{
    const long minsize = (min_target - st->minmax_reservoir + 7) / 8;
    if(choice >= NB) choice = NB - 1;
    natural = (bits[choice] + 7) / 8;
    *bytes = minsize > natural ? minsize : natural;
  }
  if(*bytes < natural) branches[4]++;
  if(*bytes > natural) branches[5]++;
  this_bits = *bytes * 8;

  if(B->min_bitsper > 0 || B->max_bitsper > 0){
    if(max_target > 0 && this_bits > max_target) st->minmax_reservoir += this_bits - max_target;
    else if(min_target > 0 && this_bits < min_target) st->minmax_reservoir += this_bits - min_target;
    else if(st->minmax_reservoir > B->desired_fill){
      if(max_target > 0){
        st->minmax_reservoir += this_bits - max_target;
        if(st->minmax_reservoir < B->desired_fill) st->minmax_reservoir = B->desired_fill;
      }else st->minmax_reservoir = B->desired_fill;
    }else{
      if(min_target > 0){
        st->minmax_reservoir += this_bits - min_target;
        if(st->minmax_reservoir > B->desired_fill) st->minmax_reservoir = B->desired_fill;
      }else st->minmax_reservoir = B->desired_fill;
    }
  }
  if(B->avg_bitsper > 0) st->avg_reservoir += this_bits - avg_target;
  st->choice = choice;
  return choice;
}

/* nblocks blocks of one stream from *state (NULL: vorbis_bitrate_init's state): W [nblocks], bits [nblocks][NB];
 * choice / bytes [nblocks]; after [nblocks] the state after every block (may be NULL); branches [VBO_BR_BRANCHES]
 * accumulated.  Returns 0, or -1 for an un-managed info. */
int vbo_bitrate_run(const vb200_bitrate_info *bi, long rate, int bs0, int bs1, int nblocks, const int *W,
                    const int *bits, vb200_bitrate_state *state, int *choice, long *bytes, vb200_bitrate_state *after,
                    long *branches){
  vbo_bitrate B;
  vb200_bitrate_state st;
  int k;
  if(vbo_bitrate_derive(bi, rate, bs0, bs1, &B)) return -1;
  if(state) st = *state; else vbo_bitrate_fresh(&B, &st);
  for(k = 0; k < nblocks; k++){
    choice[k] = vbo_bitrate_addblock(&B, W[k] ? 1 : 0, bits + (size_t)k * NB, &st, bytes + k, branches);
    if(after) after[k] = st;
  }
  if(state) *state = st;
  return 0;
}
