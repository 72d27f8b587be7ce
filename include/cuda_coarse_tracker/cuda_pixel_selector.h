// DSO's PixelSelector on the device (n10, include/tandem_b200.h): makeMaps (tandem/src/FullSystem/PixelSelector2.cpp:142-291)
// on a tdm_pyramid's levels 0..2, with currentPotential carried across calls.  CudaImmaturePoints::makeNewTraces runs it
// together with the ImmaturePoint constructor; INTEGRATION.md shows the call sites.  Owns one tdm_selector handle; not
// copyable.
#ifndef TDM_CUDA_PIXEL_SELECTOR_H
#define TDM_CUDA_PIXEL_SELECTOR_H

struct tdm_selector;   // include/tandem_b200.h
struct tdm_pyramid;

class CudaPixelSelector {
 public:
  // PixelSelector(w, h) with the reference's settings (util/settings.cpp:132-135); currentPotential starts at 3
  CudaPixelSelector(int w, int h, int device = 0);
  ~CudaPixelSelector();
  CudaPixelSelector(const CudaPixelSelector &) = delete;
  CudaPixelSelector &operator=(const CudaPixelSelector &) = delete;

  // makeMaps(fh, map_out, density, recursionsLeft, false, thFactor) on the pyramid of fh; map_out (w*h floats, may be null)
  // receives 0 / 1 / 2 / 4 per pixel.  Returns the number of selected pixels.  Blocking.
  int makeMaps(tdm_pyramid *pyramid, float *map_out, float density, int recursionsLeft = 1, float thFactor = 1);
  int currentPotential() const;
  void setCurrentPotential(int potential);
  tdm_selector *handle() const { return handle_; }

 private:
  tdm_selector *handle_ = nullptr;
};

#endif
