# TEST INFRASTRUCTURE ONLY: the stereo parity oracle. Nothing here is linked into, imported by, or shipped with the
# product (mrcal_b200/).
#
#   make -f stereo.mk   compile the reference's own stereo.c, where it lies under $(REF), into
#                       _ref/libmrcal_stereo_ref.so, linked against _ref/libmrcal_ref.so (the Makefile's `ref`
#                       target, built first) for the projections and pose utilities stereo.c calls. The one symbol
#                       neither provides, LAPACK's dgeev_, comes from stubs/stereo_stubs.c. No reference source is
#                       copied. Without the reference tree or libmrcal_ref.so this does nothing.
REF    ?= /root/reference
HERE   := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
OUT    := $(HERE)_ref
GEN    := $(OUT)/gen
CFLAGS_REF := -O2 -fPIC -fno-omit-frame-pointer -I$(HERE)stubs -I$(GEN) -I$(REF) -w

.PHONY: all
all: $(if $(wildcard $(REF)/stereo.c),$(if $(wildcard $(OUT)/libmrcal_ref.so),$(OUT)/libmrcal_stereo_ref.so))

$(OUT)/libmrcal_stereo_ref.so: $(REF)/stereo.c $(HERE)stubs/stereo_stubs.c $(OUT)/libmrcal_ref.so
	gcc -std=gnu11 $(CFLAGS_REF) -shared -o $@.tmp $(REF)/stereo.c $(HERE)stubs/stereo_stubs.c \
	    -L$(OUT) -l:libmrcal_ref.so -Wl,-rpath,'$$ORIGIN' -Wl,--no-undefined -lm
	mv -f $@.tmp $@
