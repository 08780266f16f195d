// TSDValueConverter's value -> tsd / weight constants now live with the rest of the 16-bit cell
// encoding in value_conversion.h.  This name stays for the refinement's CPU emulation harness
// (tests/emulation/refine2d_tsdf_emulation.cc), which includes it; product code includes
// value_conversion.h.
#ifndef CSM_TSDF_CONVERSION_H_
#define CSM_TSDF_CONVERSION_H_

#include "value_conversion.h"

#endif  // CSM_TSDF_CONVERSION_H_
