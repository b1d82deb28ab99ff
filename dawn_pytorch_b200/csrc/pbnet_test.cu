// dawn_pbnet_test_kernel (include/dawn_pbnet.h): each row kernel of the PBnet decoder (pbnet_kernels.cuh) on caller-owned device
// buffers, through the same launch functions generate uses, so the tests can hold every kernel to float64 at any accepted shape.
#include <string>

#include "../../include/dawn_pbnet.h"
#include "common.cuh"
#include "pbnet_kernels.cuh"

using namespace dawn;

namespace {

int refuse(const char* why) {
  set_last_error(std::string("pbnet test: ") + why);
  return -1;
}

}  // namespace

extern "C" int dawn_pbnet_test_kernel(const dawn_pbnet_kernel_case* c, void* stream) {
  if (!c) return refuse("null case");
  if (c->D < 32 || c->D > kPbMaxD || c->D % 32 != 0) return refuse("D must be a multiple of 32 from 32 to 256");
  cudaStream_t st = (cudaStream_t)stream;
  switch (c->kernel) {
    case DAWN_PBNET_MEMORY:
      if (!c->x || !c->z || !c->w || !c->xref || (c->PE > 0 && !c->w2) || !c->out) return refuse("memory needs x, z, w, xref, w2 and out");
      if (c->bs < 1 || c->F < 1 || (long long)c->bs * c->F > (1 << 24) || c->Lz < 1 || c->PE < 0)
        return refuse("bad memory geometry");
      DAWN_TRY(launch_pb_memory(c->x, c->z, c->Lz, c->w, c->xref, c->PE, c->w2, c->bs, c->F, c->D, c->out, st));
      break;
    case DAWN_PBNET_PROJ: {
      if (!c->x || !c->w || !c->out) return refuse("projection needs x, w and out");
      if (c->T < 1 || c->F < 1 || (c->ldx != 0 && c->ldx < c->D) || c->hid < 32 || c->hid % 32 != 0 ||
          c->hid > 32 * kPbMaxHeads || c->ngroups < 1 || c->ngroups > kPbMaxGroups || c->npairs < 0 || c->npairs > 16)
        return refuse("bad projection geometry");
      PbProjGroups g{};
      bool rotary = false;
      for (int i = 0; i < c->ngroups; ++i) {
        if (c->flags[i] & ~(PB_SCALE | PB_ROTARY)) return refuse("projection flags are PB_SCALE (1) | PB_ROTARY (2)");
        g.flags[i] = c->flags[i];
        rotary = rotary || (c->flags[i] & PB_ROTARY);
      }
      if (rotary && (c->npairs < 1 || !c->rot)) return refuse("a rotary group needs rot and npairs >= 1");
      DAWN_TRY(launch_pb_proj(c->x, c->ldx, c->T, c->F, c->D, c->w, c->hid, c->ngroups, g, c->qscale, c->rot, c->npairs, c->out, st));
      break;
    }
    case DAWN_PBNET_OUT_LN:
      if (!c->x || !c->w || !c->res || !c->gamma || !c->beta || !c->out)
        return refuse("out + LayerNorm needs x, w, res, gamma, beta and out");
      if (c->T < 1 || c->hid < 32 || c->hid % 32 != 0 || c->hid > 32 * kPbMaxHeads || (c->ldr != 0 && c->ldr < c->D))
        return refuse("bad out + LayerNorm geometry");
      DAWN_TRY(launch_pb_out_ln(c->x, c->hid, c->w, c->res, c->ldr, c->gamma, c->beta, c->T, c->D, c->out, st));
      break;
    case DAWN_PBNET_FFN_LN:
      if (!c->x || !c->w || !c->b1 || !c->w2 || !c->b2 || !c->gamma || !c->beta) return refuse("FFN needs x, w, b1, w2, b2, gamma and beta");
      if (c->T < 1 || c->ff < 1 || c->ff > kPbMaxFF) return refuse("bad FFN geometry");
      if (c->wf && (!c->bf || !c->mask || !c->out || c->nout < 1 || c->nout > kPbMaxOut))
        return refuse("finallayer needs bf, mask, out and 1 to 32 outputs");
      DAWN_TRY(launch_pb_ffn_ln(c->x, c->T, c->D, c->w, c->b1, c->ff, c->w2, c->b2, c->gamma, c->beta, c->wf, c->wf ? c->bf : nullptr,
                                c->nout, c->mask, c->out, st));
      break;
    default:
      return refuse("unknown kernel");
  }
  DAWN_CUDA_OK(cudaStreamSynchronize(st));
  return 0;
}
