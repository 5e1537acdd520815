# Build of the H100-native volrend backend.  No GPU is needed to build (nvcc cross-compiles).
#   make lib      volrend_b200/libvolrend_b200.so   the product: C-ABI + sm_90a kernels
#   make oracle   oracle/liboracle.so               CPU restatement (test infrastructure), and
#                 oracle/libprobe_oracle.so         the same with the probe disc
#                 oracle/libweights_oracle.so       ... with the leaf-weights pass
#                 oracle/libgrads_oracle.so         ... with the leaf-gradient pass
#                 oracle/liberror_oracle.so         ... with the leaf-error pass
#                 oracle/libsurface_harness.so      cudaArray + surface objects for the surface render path's tests
#   make ref      oracle/_ref/*                     the unmodified reference (+ its gen_wireframe, probe and mesh harnesses), built from
#                                                   $(VOLREND_REF) (only when it exists)
#   make shim     oracle/_ref/volrend_headless ...  reference CLI linked against OUR backend
NVCC      ?= nvcc
CXX       ?= g++
CC        ?= gcc
ARCH      := -gencode arch=compute_90a,code=sm_90a
NVFLAGS   := $(ARCH) -O3 -std=c++17 -lineinfo -Xcompiler -fPIC -Iinclude -Ivolrend_b200/csrc \
             -diag-suppress 20012
OBJ       := build/obj
KBDS      := m1 1 4 9 16 25
KOBJS     := $(foreach k,$(KBDS),$(OBJ)/vr_kernels_$(k).o)
LIB       := volrend_b200/libvolrend_b200.so
VOLREND_REF ?= /root/reference

.PHONY: all lib oracle ref shim clean
all: lib oracle

lib: $(LIB)

$(OBJ)/vr_kernels_m1.o: volrend_b200/csrc/vr_kernels_inst.cu volrend_b200/csrc/vr_march.cuh volrend_b200/csrc/vr_march_q.cuh volrend_b200/csrc/vr_types.h volrend_b200/csrc/vr_kernels.h include/volrend_b200.h
	@mkdir -p $(OBJ)
	$(NVCC) $(NVFLAGS) -DVR_KBD=-1 -Xptxas -v -c $< -o $@ 2> $(OBJ)/ptxas_m1.log || (cat $(OBJ)/ptxas_m1.log; false)

$(OBJ)/vr_kernels_%.o: volrend_b200/csrc/vr_kernels_inst.cu volrend_b200/csrc/vr_march.cuh volrend_b200/csrc/vr_march_q.cuh volrend_b200/csrc/vr_types.h volrend_b200/csrc/vr_kernels.h include/volrend_b200.h
	@mkdir -p $(OBJ)
	$(NVCC) $(NVFLAGS) -DVR_KBD=$* -Xptxas -v -c $< -o $@ 2> $(OBJ)/ptxas_$*.log || (cat $(OBJ)/ptxas_$*.log; false)

$(OBJ)/vr_api.o: volrend_b200/csrc/vr_api.cu volrend_b200/csrc/vr_tree.h volrend_b200/csrc/vr_frames.h volrend_b200/csrc/vr_types.h volrend_b200/csrc/vr_kernels.h volrend_b200/csrc/vr_raster.h volrend_b200/csrc/vr_wire.h volrend_b200/csrc/vr_probe.h volrend_b200/csrc/vr_normals.h volrend_b200/csrc/vr_quant.h volrend_b200/csrc/vr_query.h volrend_b200/csrc/vr_tv.h volrend_b200/csrc/vr_build.h volrend_b200/csrc/vr_ssim.h volrend_b200/csrc/vr_iso.h include/volrend_b200.h
	@mkdir -p $(OBJ)
	$(NVCC) $(NVFLAGS) -c $< -o $@

$(OBJ)/vr_tree.o: volrend_b200/csrc/vr_tree.cu volrend_b200/csrc/vr_tree.h volrend_b200/csrc/vr_frames.h volrend_b200/csrc/vr_types.h volrend_b200/csrc/vr_kernels.h volrend_b200/csrc/vr_wire.h include/volrend_b200.h
	@mkdir -p $(OBJ)
	$(NVCC) $(NVFLAGS) -Xptxas -v -c $< -o $@ 2> $(OBJ)/ptxas_tree.log || (cat $(OBJ)/ptxas_tree.log; false)

$(OBJ)/vr_cull.o: volrend_b200/csrc/vr_cull.cu volrend_b200/csrc/vr_tree.h volrend_b200/csrc/vr_march.cuh volrend_b200/csrc/vr_types.h volrend_b200/csrc/vr_frames.h volrend_b200/csrc/vr_wire.h include/volrend_b200.h
	@mkdir -p $(OBJ)
	$(NVCC) $(NVFLAGS) -Xptxas -v -c $< -o $@ 2> $(OBJ)/ptxas_cull.log || (cat $(OBJ)/ptxas_cull.log; false)

$(OBJ)/vr_raster.o: volrend_b200/csrc/vr_raster.cu volrend_b200/csrc/vr_raster.h
	@mkdir -p $(OBJ)
	$(NVCC) $(NVFLAGS) -Xptxas -v -c $< -o $@ 2> $(OBJ)/ptxas_raster.log || (cat $(OBJ)/ptxas_raster.log; false)

$(OBJ)/vr_wire.o: volrend_b200/csrc/vr_wire.cu volrend_b200/csrc/vr_wire.h volrend_b200/csrc/vr_wire_walk.cuh volrend_b200/csrc/vr_types.h
	@mkdir -p $(OBJ)
	$(NVCC) $(NVFLAGS) -Xptxas -v -c $< -o $@ 2> $(OBJ)/ptxas_wire.log || (cat $(OBJ)/ptxas_wire.log; false)

$(OBJ)/vr_tv.o: volrend_b200/csrc/vr_tv.cu volrend_b200/csrc/vr_tv.h volrend_b200/csrc/vr_wire_walk.cuh volrend_b200/csrc/vr_wire.h volrend_b200/csrc/vr_probe.h volrend_b200/csrc/vr_types.h include/volrend_b200.h
	@mkdir -p $(OBJ)
	$(NVCC) $(NVFLAGS) -Xptxas -v -c $< -o $@ 2> $(OBJ)/ptxas_tv.log || (cat $(OBJ)/ptxas_tv.log; false)

$(OBJ)/vr_ssim.o: volrend_b200/csrc/vr_ssim.cu volrend_b200/csrc/vr_ssim.h
	@mkdir -p $(OBJ)
	$(NVCC) $(NVFLAGS) -Xptxas -v -c $< -o $@ 2> $(OBJ)/ptxas_ssim.log || (cat $(OBJ)/ptxas_ssim.log; false)

$(OBJ)/vr_normals.o: volrend_b200/csrc/vr_normals.cu volrend_b200/csrc/vr_normals.h volrend_b200/csrc/vr_raster.h
	@mkdir -p $(OBJ)
	$(NVCC) $(NVFLAGS) -Xptxas -v -c $< -o $@ 2> $(OBJ)/ptxas_normals.log || (cat $(OBJ)/ptxas_normals.log; false)

$(OBJ)/vr_build.o: volrend_b200/csrc/vr_build.cu volrend_b200/csrc/vr_build.h
	@mkdir -p $(OBJ)
	$(NVCC) $(NVFLAGS) -Xptxas -v -c $< -o $@ 2> $(OBJ)/ptxas_build.log || (cat $(OBJ)/ptxas_build.log; false)

$(OBJ)/vr_quant.o: volrend_b200/csrc/vr_quant.cu volrend_b200/csrc/vr_quant.h
	@mkdir -p $(OBJ)
	$(NVCC) $(NVFLAGS) -Xptxas -v -c $< -o $@ 2> $(OBJ)/ptxas_quant.log || (cat $(OBJ)/ptxas_quant.log; false)

$(OBJ)/vr_probe.o: volrend_b200/csrc/vr_probe.cu volrend_b200/csrc/vr_probe.h volrend_b200/csrc/vr_lumisphere.cuh volrend_b200/csrc/vr_march.cuh volrend_b200/csrc/vr_types.h include/volrend_b200.h
	@mkdir -p $(OBJ)
	$(NVCC) $(NVFLAGS) -Xptxas -v -c $< -o $@ 2> $(OBJ)/ptxas_probe.log || (cat $(OBJ)/ptxas_probe.log; false)

$(OBJ)/vr_query.o: volrend_b200/csrc/vr_query.cu volrend_b200/csrc/vr_query.h volrend_b200/csrc/vr_probe.h volrend_b200/csrc/vr_lumisphere.cuh volrend_b200/csrc/vr_march.cuh volrend_b200/csrc/vr_types.h include/volrend_b200.h
	@mkdir -p $(OBJ)
	$(NVCC) $(NVFLAGS) -Xptxas -v -c $< -o $@ 2> $(OBJ)/ptxas_query.log || (cat $(OBJ)/ptxas_query.log; false)

$(OBJ)/vr_iso.o: volrend_b200/csrc/vr_iso.cu volrend_b200/csrc/vr_iso.h volrend_b200/csrc/vr_iso_table.h volrend_b200/csrc/vr_probe.h volrend_b200/csrc/vr_lumisphere.cuh volrend_b200/csrc/vr_march.cuh volrend_b200/csrc/vr_types.h include/volrend_b200.h
	@mkdir -p $(OBJ)
	$(NVCC) $(NVFLAGS) -Xptxas -v -c $< -o $@ 2> $(OBJ)/ptxas_iso.log || (cat $(OBJ)/ptxas_iso.log; false)

$(OBJ)/vr_mg.o: volrend_b200/csrc/vr_mg.cu include/volrend_b200.h
	@mkdir -p $(OBJ)
	$(NVCC) $(NVFLAGS) -c $< -o $@

$(OBJ)/vr_png.o: volrend_b200/csrc/vr_png.cpp volrend_b200/csrc/vr_frames.h include/volrend_b200.h
	@mkdir -p $(OBJ)
	$(CXX) -O3 -std=c++17 -fPIC -Iinclude -c $< -o $@

$(LIB): $(OBJ)/vr_api.o $(OBJ)/vr_tree.o $(OBJ)/vr_cull.o $(OBJ)/vr_raster.o $(OBJ)/vr_wire.o $(OBJ)/vr_tv.o $(OBJ)/vr_ssim.o $(OBJ)/vr_normals.o $(OBJ)/vr_quant.o $(OBJ)/vr_build.o $(OBJ)/vr_probe.o $(OBJ)/vr_query.o $(OBJ)/vr_iso.o $(OBJ)/vr_mg.o $(OBJ)/vr_png.o $(KOBJS)
	$(NVCC) $(ARCH) -shared -o $@ $^ -lz -lpthread

oracle: oracle/liboracle.so oracle/libprobe_oracle.so oracle/libweights_oracle.so oracle/libgrads_oracle.so oracle/liberror_oracle.so oracle/libsurface_harness.so
oracle/liboracle.so: oracle/march_oracle.c oracle/march_oracle.h
	$(CC) -O2 -ffp-contract=off -fno-fast-math -fPIC -shared -pthread -o $@ $< -lm
oracle/libprobe_oracle.so: oracle/probe_oracle.c oracle/march_oracle.c oracle/march_oracle.h
	$(CC) -O2 -ffp-contract=off -fno-fast-math -fPIC -shared -pthread -o $@ $< -lm
oracle/libweights_oracle.so: oracle/weights_oracle.c oracle/march_oracle.c oracle/march_oracle.h
	$(CC) -O2 -ffp-contract=off -fno-fast-math -fPIC -shared -pthread -o $@ $< -lm
oracle/libgrads_oracle.so: oracle/grads_oracle.c oracle/march_oracle.c oracle/march_oracle.h
	$(CC) -O2 -ffp-contract=off -fno-fast-math -fPIC -shared -pthread -o $@ $< -lm
oracle/liberror_oracle.so: oracle/error_oracle.c oracle/march_oracle.c oracle/march_oracle.h
	$(CC) -O2 -ffp-contract=off -fno-fast-math -fPIC -shared -pthread -o $@ $< -lm
oracle/libsurface_harness.so: oracle/surface_harness.cu
	$(NVCC) $(ARCH) -O2 -std=c++17 -Xcompiler -fPIC -shared -o $@ $<

ref:
	@if [ -d "$(VOLREND_REF)/src/cuda" ]; then $(MAKE) -C oracle -f Makefile.ref VOLREND_REF=$(VOLREND_REF) && \
	   $(MAKE) -C oracle -f Makefile.wire VOLREND_REF=$(VOLREND_REF) && \
	   $(MAKE) -C oracle -f Makefile.probe VOLREND_REF=$(VOLREND_REF) && \
	   $(MAKE) -C oracle -f Makefile.query VOLREND_REF=$(VOLREND_REF) && \
	   $(MAKE) -C oracle -f Makefile.mesh VOLREND_REF=$(VOLREND_REF); \
	 else echo "reference tree $(VOLREND_REF) not present: using prebuilt oracle/_ref if any"; fi

shim:
	@if [ -d "$(VOLREND_REF)/src/cuda" ]; then $(MAKE) -C volrend_b200/csrc/shim VOLREND_REF=$(VOLREND_REF); \
	 else echo "reference tree $(VOLREND_REF) not present: shim needs the reference headers"; fi

clean:
	rm -rf build $(LIB) oracle/liboracle.so oracle/libprobe_oracle.so oracle/libweights_oracle.so oracle/libgrads_oracle.so oracle/liberror_oracle.so oracle/libsurface_harness.so oracle/_ref
