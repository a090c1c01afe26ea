/* vb200_vorbis_setup.h — libvorbis' modes, floors and residues as the library's structs, for the host bindings
 * (vb200_decode.c, vb200_mapping0.c, vb200_ref_shim.c).  Static inline functions in a header, so that a library
 * linking one of those files needs no other object.  Included after codec_internal.h and vorbis_b200.h.  Each caller
 * keeps its own refusals: these functions only say what the structs cannot describe.
 */
#ifndef VB200_VORBIS_SETUP_H
#define VB200_VORBIS_SETUP_H

#include "misc.h"

/* the mapping of mode w where the modes are the two of block flags 0 and 1 on mappings of type 0 with at most
 * VB200_MAX_SUBMAPS submaps, else NULL */
static inline vorbis_info_mapping0 *vb200vs_mapping(const codec_setup_info *ci, int w){
  vorbis_info_mapping0 *mp;
  if(ci->modes != 2 || ci->mode_param[w]->blockflag != w || ci->map_type[ci->mode_param[w]->mapping] != 0) return NULL;
  mp = (vorbis_info_mapping0*)ci->map_param[ci->mode_param[w]->mapping];
  return mp->submaps > VB200_MAX_SUBMAPS ? NULL : mp;
}

/* the floor-1 curve of one submap */
static inline void vb200vs_floor1(vb200_floor1_setup *o, const vorbis_info_floor1 *fi, const vorbis_look_floor1 *lk){
  int k;
  o->posts = lk->posts;
  for(k = 0; k < lk->posts; k++) o->postlist[k] = fi->postlist[k];
  o->mult = fi->mult; o->n = lk->n;
  o->maxover = fi->maxover; o->maxunder = fi->maxunder; o->maxerr = fi->maxerr;
  o->twofitweight = fi->twofitweight; o->twofitatten = fi->twofitatten;
}

/* The floor and residue fields of both modes' submaps (residue type -1 past a mode's submaps), the stage books laid
 * out as res0_look lays out partbooks (lib/res0.c:274-292) and partvals = partitions ^ dim(groupbook) as res0_look
 * counts look->partvals (:295-297).  dim: the dimension of the caller's book 0, dim_stride: the bytes from one book's
 * dimension to the next.  0, or OV_EIMPL where a mode is not one vb200vs_mapping takes. */
static inline int vb200vs_entropy(const codec_setup_info *ci, const int32_t *dim, size_t dim_stride,
                                  vb200_floor_decode floor[2][VB200_MAX_SUBMAPS],
                                  vb200_residue_decode residue[2][VB200_MAX_SUBMAPS]){
  int w, j, k, c;
  for(w = 0; w < 2; w++){
    const vorbis_info_mapping0 *mp = vb200vs_mapping(ci, w);
    if(!mp) return OV_EIMPL;
    for(j = 0; j < VB200_MAX_SUBMAPS; j++) residue[w][j].type = -1;
    for(j = 0; j < mp->submaps; j++){
      const int fl = mp->floorsubmap[j], rs = mp->residuesubmap[j];
      const vorbis_info_residue0 *ri = (const vorbis_info_residue0*)ci->residue_param[rs];
      const int32_t groupdim = *(const int32_t*)((const char*)dim + dim_stride * ri->groupbook);
      vb200_floor_decode *f = &floor[w][j];
      vb200_residue_decode *r = &residue[w][j];
      int acc = 0;
      f->type = ci->floor_type[fl];
      if(f->type == 1){
        const vorbis_info_floor1 *fi = (const vorbis_info_floor1*)ci->floor_param[fl];
        f->partitions = fi->partitions;
        for(k = 0; k < fi->partitions && k < 31; k++) f->partitionclass[k] = fi->partitionclass[k];
        for(k = 0; k < 16; k++){
          int s;
          f->class_dim[k] = fi->class_dim[k]; f->class_subs[k] = fi->class_subs[k]; f->class_book[k] = fi->class_book[k];
          for(s = 0; s < 8; s++) f->class_subbook[k][s] = fi->class_subbook[k][s];
        }
      }
      r->type = ci->residue_type[rs];
      r->begin = (int32_t)ri->begin; r->end = (int32_t)ri->end; r->grouping = ri->grouping;
      r->partitions = ri->partitions; r->groupbook = ri->groupbook;
      r->partvals = 1;
      for(k = 0; k < groupdim; k++) r->partvals *= ri->partitions;
      for(c = 0; c < 64; c++){
        const int stages = c < ri->partitions ? ov_ilog((ogg_uint32_t)ri->secondstages[c]) : 0;
        for(k = 0; k < 8; k++)
          r->stagebook[c][k] = k < stages && (ri->secondstages[c] & (1 << k)) ? ri->booklist[acc++] : -1;
      }
    }
  }
  return 0;
}

#endif
