# Test-only builds for the SIFT extractor (nothing here is on the product path):
#  * _build/libsift_emul.so  host build of the SIFT CUDA path's functors (see sift_emul.cpp), g++ -ffp-contract=off;
#  * _ref/sift_ref.py        the UNMODIFIED reference SIFT extractor file.
# The reference copy next to the reference matcher copy of the Makefile here,
# as _ref/sift_ref.py (git-ignored, like the rest of _ref/).  It needs cv2 and is loaded with stand-ins by
# sift_ref_loader.py, for the fixture generator make_golden_sift.py, tests/test_sift_oracle_golden.py and the reference
# leg of tools/sift_bench.py.  The reference directory is the one the Makefile's REF_SRC names; nothing is copied where
# it does not exist.
#   make -C oracle -f sift_ref.mk
include Makefile
.DEFAULT_GOAL := sift-all
SIFT_EMUL := _build/libsift_emul.so
SIFT_SRC := $(dir $(REF_SRC))sift.py
SIFT_REF := _ref/sift_ref.py

sift-all: $(SIFT_EMUL) sift-ref

$(SIFT_EMUL): sift_emul.cpp ../lightglue_b200/csrc/sift_pipeline.h
	@mkdir -p _build
	$(CXX) -O2 -std=c++17 -fPIC -shared -pthread -ffp-contract=off -o $@ sift_emul.cpp -lm

sift-ref:
	@if [ -f $(SIFT_SRC) ]; then mkdir -p _ref && cp -u --no-preserve=mode $(SIFT_SRC) $(SIFT_REF); fi

.PHONY: sift-all sift-ref
