# TEST INFRASTRUCTURE ONLY -- the reference harness of the custom-node fixture
# (sims/customnodes), built with the flags, shims and reference library of
# oracle/Makefile by its generic harness rule:
#     make -C oracle -f customnodes.mk customnodes
include Makefile

customnodes: $(OUT)/ref_customnodes

.PHONY: customnodes
