# Test-only: copies the UNMODIFIED reference ALIKED extractor file next to the reference matcher copy of the Makefile
# here, as _ref/aliked_ref.py (git-ignored, like the rest of _ref/).  It needs torchvision and is loaded with stand-ins by
# aliked_ref_loader.py, for the fixture generator make_golden_aliked.py and the reference leg of tools/aliked_bench.py.
# The reference directory is the one the Makefile's REF_SRC names; nothing is copied where it does not exist.
#   make -C oracle -f aliked_ref.mk
include Makefile
.DEFAULT_GOAL := aliked-ref
ALIKED_SRC := $(dir $(REF_SRC))aliked.py
ALIKED_REF := _ref/aliked_ref.py

aliked-ref:
	@if [ -f $(ALIKED_SRC) ]; then mkdir -p _ref && cp -u --no-preserve=mode $(ALIKED_SRC) $(ALIKED_REF); fi

.PHONY: aliked-ref
