#!/bin/sh
# TEST INFRASTRUCTURE -- compiles the reference's SDF CUDA kernel UNCHANGED, from where it lies under the reference
# checkout, into oracle/_ref/libsdf_refcuda.so (git-ignored; travels to the GPU box with gpurun).  The only things
# added are the <ATen/ATen.h> stand-in (oracle/refshim) and the C entry point (oracle/ref_sdf_wrap.cu).
# nvcc defaults (-O3 device code, --fmad=true) = what torch.utils.cpp_extension passes for the reference's setup.py
# (CUDA_FLAGS = [] at sdf/setup.py:5); the arch is this box's.
set -e
HERE="$(cd "$(dirname "$0")" && pwd)"
REF="${MVS_REFERENCE_ROOT:-/root/reference}"
SRC="$REF/sdf/sdf/csrc/sdf_cuda_kernel.cu"
[ -f "$SRC" ] || { echo "reference SDF kernel not found at $SRC" >&2; exit 3; }
mkdir -p "$HERE/_ref"
NVCC="${NVCC:-/usr/local/cuda/bin/nvcc}"
"$NVCC" -gencode arch=compute_90a,code=sm_90a -std=c++17 -shared -Xcompiler -fPIC -I "$HERE/refshim" \
    -o "$HERE/_ref/libsdf_refcuda.so" "$SRC" "$HERE/ref_sdf_wrap.cu"
sha256sum "$SRC" | cut -d' ' -f1 > "$HERE/_ref/sdf_cuda_kernel.sha256"
echo "$HERE/_ref/libsdf_refcuda.so"
