# Test-only copy of the UNMODIFIED reference DoG-HardNet extractor file (nothing here is on the product path):
#  * _ref/dog_hardnet_ref.py  lightglue/dog_hardnet.py, next to _ref/sift_ref.py (sift_ref.mk), which it imports.
# It needs kornia and is loaded with the stand-ins of oracle/doghardnet_oracle.py by doghardnet_ref_loader.py.  Copied
# only when the reference directory the Makefile's REF_SRC names exists.
#   make -C oracle -f doghardnet_ref.mk
include Makefile
.DEFAULT_GOAL := dhn-ref
DHN_SRC := $(dir $(REF_SRC))dog_hardnet.py
DHN_REF := _ref/dog_hardnet_ref.py

dhn-ref:
	@if [ -f $(DHN_SRC) ]; then mkdir -p _ref && cp -u --no-preserve=mode $(DHN_SRC) $(DHN_REF); fi

.PHONY: dhn-ref
