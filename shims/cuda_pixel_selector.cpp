// CudaPixelSelector over the tandem_b200 C ABI.  Errors throw std::runtime_error, as the tracker shim's do.
#include "cuda_coarse_tracker/cuda_pixel_selector.h"

#include <stdexcept>
#include <string>

#include "tandem_b200.h"

static void chk(int rc, const char *where) {
  if (rc != TDM_OK) throw std::runtime_error(std::string(where) + ": " + tdm_last_error());
}

CudaPixelSelector::CudaPixelSelector(int w, int h, int device) {
  chk(tdm_selector_create(w, h, nullptr, device, &handle_), "CudaPixelSelector");
}

CudaPixelSelector::~CudaPixelSelector() { tdm_selector_destroy(handle_); }

int CudaPixelSelector::makeMaps(tdm_pyramid *pyramid, float *map_out, float density, int recursionsLeft, float thFactor) {
  tdm_select_result r;
  chk(tdm_selector_make_maps(handle_, pyramid, density, recursionsLeft, thFactor, map_out, &r), "CudaPixelSelector::makeMaps");
  return r.num_selected;
}

int CudaPixelSelector::currentPotential() const {
  int p = 0;
  chk(tdm_selector_get_potential(handle_, &p), "CudaPixelSelector::currentPotential");
  return p;
}

void CudaPixelSelector::setCurrentPotential(int potential) {
  chk(tdm_selector_set_potential(handle_, potential), "CudaPixelSelector::setCurrentPotential");
}
