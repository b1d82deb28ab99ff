/* dawn_video.h — C-ABI of the video generator's pixel stages that are not part of a network.
 *
 * dawn_portrait_resize: the portrait preparation of unified_video_generator.py:320-325 and 372 on the device:
 * `transforms.Resize((S, S))` of a PIL RGB image (Pillow's 8-bit bilinear resampler, `Image.resize((S, S), Image.BILINEAR)`,
 * bit for bit), `ToTensor` (u / 255), `* 255` and `/ 255.`, all in fp32 as torch computes them on the host.
 *   img      (H0, W0, 3) uint8 RGB on the device, 1 <= H0, W0 <= 8192
 *   S        output side, 1 <= S <= 8192
 *   source   (3, S, S) fp32 on the device: what the LFG decoder and the UNet's source features take
 *   resized  (S, S, 3) uint8 on the device: the resized image itself, or NULL
 * The resampling coefficients are computed on the host in double precision, as Pillow does, converted to 22-bit fixed point,
 * uploaded on `stream` and freed with the stream's work; the only host wait is the upload of that table.  Pillow's two passes are
 * kept: the horizontal one over the rows the vertical one reads, into a uint8 image, then the vertical one; a pass is skipped
 * exactly when Pillow skips it (that axis keeps its size).
 * Return: 0 ok, -1 bad argument (message through dawn_last_error, declared in include/dawn_unet.h), -2 CUDA error.
 */
#ifndef DAWN_VIDEO_H_
#define DAWN_VIDEO_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

int dawn_portrait_resize(const uint8_t* img, int H0, int W0, int S, float* source, uint8_t* resized, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DAWN_VIDEO_H_ */
