// Device pre-processing (see preproc.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace lm {
// per slice: body mask on the 128x128 thumbnail -> crop box [r0,c0,r1,c1) (int32 x4 per slice);
// mask_out (optional, may be nullptr): the full-resolution 0/1 body mask (S,H,W).
int launch_bodymask(const int16_t* vol, int S, int H, int W, int32_t* boxes, uint8_t* mask_out, int num_sms,
                    cudaStream_t stream);
// (optionally clip to [-1024,600] HU,) crop to the box, bilinear zoom to OHxOW in float64, round half away from zero.
int launch_resize(const int16_t* vol, int S, int H, int W, const int32_t* boxes, int16_t* out, int OH, int OW, int clip,
                  int num_sms, cudaStream_t stream);
// Float volumes (float32 / float64 HU; the reference keeps the dtype through its pre-processing, utils.py:44-45,108-110):
// same body mask, the resize leaves the interpolated value unrounded and writes the NORMALISED fp32 network input
// ((x + 1024) / 1624 evaluated in the volume's dtype, mask.py:167-168,178-182).
int launch_bodymask_float(const void* vol, int is_f64, int S, int H, int W, int32_t* boxes, uint8_t* mask_out, int num_sms,
                          cudaStream_t stream);
int launch_resize_float(const void* vol, int is_f64, int S, int H, int W, const int32_t* boxes, float* out_norm, int OH, int OW,
                        int num_sms, cudaStream_t stream);
// Native orientation <-> LPS (axis permutation + flips, see preproc.cu orient_kernel): dims_lps = shape of the LPS array,
// lps = transpose(native, perm) flipped along every axis k with flip[k].  to_lps = 1: native -> LPS; 0: LPS -> native.
int launch_orient_u8(const uint8_t* src, uint8_t* dst, const int dims_lps[3], const int perm[3], const int flip[3], int to_lps,
                     int num_sms, cudaStream_t stream);
// Native -> LPS in one pass with the element conversion of lm_apply_dev: src of element type `dtype` (LM_DTYPE_*);
// dst int16 for LM_DTYPE_I16 and the integer codes (clipped to [-1024, 600] unless already int16), float32 for
// LM_DTYPE_F32 / F16 / BF16, float64 for LM_DTYPE_F64.  Returns -1 for an unknown code.
int launch_orient_convert(const void* src, int dtype, void* dst, const int dims_lps[3], const int perm[3], const int flip[3],
                          int num_sms, cudaStream_t stream);

// Axis permutation + flips between an array in its native orientation and the LPS array the path works on
// (sitk.DICOMOrient, mask.py:157-164,204-208; lungmask_b200/orient.py states the index map):
//   lps[i0][i1][i2] = native[c],  c[perm[k]] = flip[k] ? dims_lps[k] - 1 - i_k : i_k.
struct OrientMap { int dl[3]; int perm[3]; int flip[3]; };
#ifdef __CUDACC__
// The LPS index i of the native-orientation voxel t (row-major over the native dims dn, dn[perm[k]] = dl[k]).
__device__ __forceinline__ void orient_lps_of_native(const OrientMap& m, const int dn[3], size_t t, int i[3]) {
  int c[3];
  c[2] = (int)(t % dn[2]);
  c[1] = (int)((t / dn[2]) % dn[1]);
  c[0] = (int)(t / ((size_t)dn[2] * dn[1]));
  for (int k = 0; k < 3; ++k) {
    const int ck = m.perm[k] == 0 ? c[0] : (m.perm[k] == 1 ? c[1] : c[2]);   // c[perm[k]] without a run-time array index
    i[k] = m.flip[k] ? m.dl[k] - 1 - ck : ck;
  }
}
#endif
}  // namespace lm
