#!/usr/bin/env bash
# TEST INFRASTRUCTURE ONLY -- builds the reference's own CPU implementation as the parity oracle and
# CPU baseline. Outputs go ONLY to oracle/_ref/ (git-ignored).
#
# The reference is header-only C++14 written for icpc+MKL+MPI; g++ rejects six icpc-isms, so the
# recipe stages a scratch copy of src/ and test/ under oracle/_ref/refsrc (a build artefact, never
# committed) and applies six mechanical, non-arithmetic edits (SURVEY.md Appendix B), then compiles
# two small drivers (oracle/ref_driver_*.cpp) against it with the mkl.h / mpi.h shims in oracle/shim.
# Needs the reference sources (CAPITAL_REFERENCE); where they are absent the prebuilt
# binaries in oracle/_ref/ are used as-is.
set -euo pipefail
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
REF="${CAPITAL_REFERENCE:-/root/reference}"
OUT="$HERE/_ref"
if [ ! -d "$REF/src/alg" ]; then
  if [ -x "$OUT/ref_cholinv" ] && [ -x "$OUT/ref_cacqr" ]; then echo "[oracle] $REF absent; using prebuilt $OUT"; exit 0; fi
  echo "[oracle] $REF absent and no prebuilt binaries in $OUT" >&2; exit 1
fi
SP="$(python -c 'import scipy,os;print(os.path.join(os.path.dirname(os.path.dirname(scipy.__file__)),"scipy.libs"))')"
BLAS="$(ls "$SP"/libscipy_openblas*.so | head -1)"
mkdir -p "$OUT"; rm -rf "$OUT/refsrc"; mkdir -p "$OUT/refsrc"
cp -r "$REF/src" "$REF/test" "$OUT/refsrc/"; chmod -R u+w "$OUT/refsrc"
cd "$OUT/refsrc"
# 1-3: a member alias may not re-declare a template parameter under g++
sed -i '9s/typename ScalarType = double, typename DimensionType = int64_t/typename ScalarT = double, typename DimensionT = int64_t/;
        13s/.*/  using ScalarType = ScalarT;/; 14s/.*/  using DimensionType = DimensionT;/' src/matrix/matrix.h
sed -i '16s/typename ScalarType, typename DimensionType/typename ScalarT, typename DimensionT/;
        19s/.*/    using ScalarType = ScalarT;/; 20s/.*/    using DimensionType = DimensionT;/' src/alg/cholesky/cholinv/cholinv.h
sed -i '18s/typename ScalarType, typename DimensionType, typename CholeskyInversionType/typename ScalarT, typename DimensionT, typename CholeskyInversionType/;
        21s/.*/    using ScalarType = ScalarT;/; 22s/.*/    using DimensionType = DimensionT;/' src/alg/qr/cacqr/cacqr.h
# 4: two-phase lookup into the dependent base class
sed -i 's/return _num_elems(rangeX, rangeY)/return StructurePolicy::_num_elems(rangeX, rangeY)/; s/? _offset(coordX/? StructurePolicy::_offset(coordX/' src/matrix/matrix.h
sed -i -E 's/(^|[^:_A-Za-z])(_assemble_matrix|_assemble|_copy|_distribute_random|_distribute_symmetric|_distribute_identity|_distribute_debug|_print)\(this/\1StructurePolicy::\2(this/g' src/matrix/matrix.hpp
# 5-6: typos in never-instantiated templates that g++ still parses
sed -i '231s/sizeof(T)/sizeof(ScalarType)/' src/matrix/structure.hpp
sed -i '8s/$/ U globalNumRows = Matrix.num_rows_global(); U globalNumColumns = Matrix.num_columns_global();/' src/util/util.hpp
cd "$OUT"
CXXFLAGS="-std=c++14 -O2 -w -I$HERE/shim -I$OUT/refsrc"
LDFLAGS="-L$SP -l:$(basename "$BLAS") -Wl,-rpath,$SP -lpthread"
g++ $CXXFLAGS "$HERE/ref_driver_cholinv.cpp" -o ref_cholinv $LDFLAGS
g++ $CXXFLAGS "$HERE/ref_driver_cacqr.cpp"   -o ref_cacqr   $LDFLAGS
echo "[oracle] built $OUT/ref_cholinv $OUT/ref_cacqr against $(basename "$BLAS")"
