# oracle/encode.mk -- TEST INFRASTRUCTURE ONLY (never linked by the product).
#
# oracle/_ref/liboracle_ex.so: the C restatement of the encoder-side colour stage (color_oracle_ex.c), built anywhere gcc exists.
# oracle/_ref/liboracle_encode.so: the encoder-side entry point into the unmodified reference colour stage
# (ref_encode.cc), linked against oracle/_ref/libheif_ref.so, which oracle/Makefile builds first.  Built only where the
# reference sources exist; elsewhere the library built there before is used.
REF ?= /root/reference
OUT := _ref
# the defines libheif_ref.so was compiled with (oracle/Makefile): the reference classes used here must have its layout
DEFS := -DLIBHEIF_EXPORTS -DHAVE_VISIBILITY -DENABLE_PLUGIN_LOADING=1 -DENABLE_MULTITHREADING_SUPPORT=1 -DENABLE_PARALLEL_TILE_DECODING=1 \
        -DHEIF_ENABLE_EXPERIMENTAL_FEATURES

.PHONY: all ref
all: $(OUT)/liboracle_ex.so ref
ifneq ($(wildcard $(REF)/libheif/box.cc),)
ref: $(OUT)/liboracle_encode.so
else
ref:
	@echo "reference sources absent: using prebuilt $(OUT)/liboracle_encode.so if any"
endif

$(OUT)/liboracle_ex.so: color_oracle_ex.c color_oracle.c
	@mkdir -p $(OUT)
	$(CC) -O2 -fPIC -shared -std=gnu11 -Wall -Wno-unused-function -ffp-contract=off -o $@ color_oracle_ex.c -ldl -lm

$(OUT)/liboracle_encode.so: ref_encode.cc $(OUT)/libheif_ref.so
	$(CXX) $(DEFS) -std=c++20 -O2 -fPIC -shared -w -I$(OUT)/include -I$(OUT)/include/libheif -I$(REF)/libheif -I$(REF)/libheif/api -o $@ ref_encode.cc \
	    -L$(OUT) -lheif_ref -Wl,-rpath,'$$ORIGIN'
