# TEST INFRASTRUCTURE ONLY.  Builds oracle/_ref/sgbm: the reference's `sgbm` matcher (3rdparty/sgbm: OpenCV 2's
# StereoSGBM + its wrapper sgbm.cpp), the UNMODIFIED sources compiled where they lie under $(SREF) (never copied into this
# repo).  __graft_entry__.build() runs it next to oracle/Makefile:  make -C oracle -f sgbm.mk
#
# Harness-side only: an empty <sys/sysctl.h> (shim/sys; glibc dropped the header that parallel.cpp includes) and the
# reference's c/iio.c without the image libraries (PFM I/O) and with the iio_save_image_float name, in place of
# 3rdparty/sgbm/iio.c, which needs png.h.  -march=x86-64-v3 instead of native, as in oracle/Makefile, so that the binary
# built in this container also runs on the GPU box's host CPU.  Run it with MALLOC_PERTURB_=255: the crop trick of sgbm.cpp
# pastes the images into Mats whose margins are never initialised, and that setting makes them zero (DESIGN.md section 4).

CC    := gcc
CXX   := g++
SREF  ?= /root/reference/3rdparty/sgbm
CREF  ?= /root/reference/c
OUT   := _ref
MARCH ?= -march=x86-64-v3
SSRC  := sgbm stereosgbm alloc arithm array convert copy datastructs gpumat lapack mathfuncs matmul matop matrix \
         opengl_interop opengl_interop_deprecated parallel persistence stat system tables_core smooth tables_imgproc

.PHONY: all
ifneq ($(wildcard $(SREF)/stereosgbm.cpp),)
all: $(OUT)/sgbm
else
all:
	@echo "oracle: $(SREF) absent -- using a prebuilt $(OUT)/sgbm if present"
endif

$(OUT)/sgbm_o:
	mkdir -p $@
$(OUT)/sgbm_o/%.o: $(SREF)/%.cpp shim/sys/sysctl.h | $(OUT)/sgbm_o
	$(CXX) -O3 $(MARCH) -w -Ishim -I$(SREF) -c $< -o $@
$(OUT)/sgbm_o/iio.o: $(CREF)/iio.c | $(OUT)/sgbm_o
	$(CC) -O3 $(MARCH) -std=gnu99 -w -DIIO_DISABLE_IMGLIBS -DIIO_USE_INCONSISTENT_NAMES -c $< -o $@
$(OUT)/sgbm: $(addprefix $(OUT)/sgbm_o/,$(addsuffix .o,$(SSRC))) $(OUT)/sgbm_o/iio.o
	$(CXX) -o $@ $^ -lm -lz
