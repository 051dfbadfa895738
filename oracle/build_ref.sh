#!/usr/bin/env bash
# TEST INFRASTRUCTURE ONLY -- builds the UNMODIFIED reference PopSift, from the
# sources where they lie ($POPSIFT_REFERENCE, default /root/reference), into
# oracle/_ref/ (git-ignored).  Nothing of the product links to it.
#
#   oracle/_ref/libpopsift_ref.so   reference library, SASS for sm_90 (+PTX)
#   oracle/_ref/ref_dump            our driver (oracle/ref_driver.cpp) over the
#                                   reference's public API (PopSift/enqueue/get)
#
# File list = /root/reference/src/CMakeLists.txt:1-40 ; flags follow
# /root/reference/CMakeLists.txt:107,150 (-rdc, --default-stream legacy).
# The reference's own build system (cmake + Boost) is NOT used.
set -euo pipefail
HERE="$(cd "$(dirname "$0")" && pwd)"
REF="${POPSIFT_REFERENCE:-/root/reference}"
OUT="$HERE/_ref"
GEN="$OUT/gen"
if [ ! -d "$REF/src/popsift" ]; then
    echo "build_ref: $REF not present (GPU box?) - using prebuilt files in $OUT" >&2
    exit 0
fi
mkdir -p "$GEN/popsift"
# sift_config.h / version.hpp are cmake-generated in the reference build
# (cmake/sift_config.h.in, cmake/version.hpp.in); written here by hand.
cat > "$GEN/popsift/sift_config.h" <<'EOC'
#pragma once
#define POPSIFT_IS_DEFINED(F) F() == 1
#define POPSIFT_HAVE_SHFL_DOWN_SYNC() 1
#define POPSIFT_HAVE_NORMF()          0
#define POPSIFT_DISABLE_GRID_FILTER() 0
#define POPSIFT_USE_NVTX()            0
EOC
cp "$GEN/popsift/sift_config.h" "$GEN/sift_config.h"
cat > "$GEN/popsift/version.hpp" <<'EOC'
#pragma once
#define POPSIFT_VERSION_MAJOR 1
#define POPSIFT_VERSION_MINOR 0
#define POPSIFT_VERSION_PATCH 0
#define POPSIFT_VERSION_STRING "1.0.0-ref"
EOC
S="$REF/src/popsift"
SRCS="$S/popsift.cpp $S/features.cu $S/sift_constants.cu $S/sift_conf.cu $S/gauss_filter.cu
 $S/s_image.cu $S/sift_pyramid.cu $S/sift_octave.cu $S/s_pyramid_build.cu $S/s_pyramid_build_aa.cu
 $S/s_pyramid_build_ai.cu $S/s_pyramid_build_ra.cu $S/s_pyramid_fixed.cu $S/sift_extremum.cu
 $S/s_extrema.cu $S/s_orientation.cu $S/s_filtergrid.cu $S/sift_desc.cu $S/s_desc_loop.cu
 $S/s_desc_iloop.cu $S/s_desc_grid.cu $S/s_desc_igrid.cu $S/s_desc_notile.cu
 $S/common/assist.cu $S/common/plane_2d.cu $S/common/write_plane_2d.cu
 $S/common/debug_macros.cu $S/common/device_prop.cu"
ARCH="-gencode arch=compute_90,code=sm_90 -gencode arch=compute_90,code=compute_90"
FLAGS="-std=c++17 -O3 -rdc=true --default-stream legacy -DCCCL_DISABLE_NVTX -DNVTX_DISABLE -w"
INC="-I$REF/src -I$GEN -I$GEN/popsift"
# a library built with other flags (another architecture) is rebuilt: the stamp records the flags it was built with
STAMP="$OUT/libpopsift_ref.flags"
if [ ! -f "$OUT/libpopsift_ref.so" ] || [ "${FORCE:-0}" = 1 ] || [ "$(cat "$STAMP" 2>/dev/null)" != "$FLAGS $ARCH" ]; then
    echo "build_ref: compiling reference library (about 1-2 min)" >&2
    rm -f "$STAMP"
    nvcc $FLAGS -x cu $ARCH -Xcompiler -fPIC -shared $INC -o "$OUT/libpopsift_ref.so" $SRCS -lcudadevrt
    printf '%s' "$FLAGS $ARCH" > "$STAMP"
fi
nvcc -std=c++17 -O2 $ARCH $INC -o "$OUT/ref_dump" "$HERE/ref_driver.cpp" \
     -L"$OUT" -lpopsift_ref -Xlinker -rpath -Xlinker '$ORIGIN' -lpthread
echo "build_ref: ok -> $OUT" >&2
