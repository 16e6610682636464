# Oracle recipe for the Plenoxels comparator (TEST / BENCH INFRASTRUCTURE, never linked into the product library):
#
#   make -f svox.mk ref   -> _ref/libref_svox.so : the reference's contrib/plenoxel volume_render_cuvol_fused.h, loss_kernel.h and
#                            misc_kernel.h compiled where they lie under $(NGP_REF) (read-only) for sm_90a, through three launcher shims
#                            and the Jittor stubs of ref_shim/stub (var.h, op.h).  Outputs only into _ref/ (git-ignored).
NGP_REF ?= /root/reference
SVOX_H  := $(NGP_REF)/contrib/plenoxel/python/jnerf/ops/svox_ops/op/op_header
NVCC    ?= nvcc
NVFLAGS := -O2 -std=c++17 --expt-relaxed-constexpr -Xcompiler -fPIC -w
GPUARCH := -gencode arch=compute_90a,code=sm_90a
SHIMS   := ref_shim/ref_svox_render.cu ref_shim/ref_svox_loss.cu ref_shim/ref_svox_misc.cu

.PHONY: ref
ref:
	@if [ -d "$(SVOX_H)" ]; then $(MAKE) -f svox.mk _ref/libref_svox.so; else echo "[oracle] $(SVOX_H) absent: keeping prebuilt _ref/ (if any)"; fi

_ref/libref_svox.so: $(SHIMS) ref_shim/stub/var.h ref_shim/stub/op.h
	@mkdir -p _ref/svox
	$(NVCC) $(GPUARCH) $(NVFLAGS) -I ref_shim/stub -I $(SVOX_H) -c ref_shim/ref_svox_render.cu -o _ref/svox/render.o
	$(NVCC) $(GPUARCH) $(NVFLAGS) -I ref_shim/stub -I $(SVOX_H) -c ref_shim/ref_svox_loss.cu -o _ref/svox/loss.o
	$(NVCC) $(GPUARCH) $(NVFLAGS) -I ref_shim/stub -I $(SVOX_H) -c ref_shim/ref_svox_misc.cu -o _ref/svox/misc.o
	$(NVCC) $(GPUARCH) -shared -o $@ _ref/svox/render.o _ref/svox/loss.o _ref/svox/misc.o
