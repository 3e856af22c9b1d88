# TEST INFRASTRUCTURE ONLY -- the reference harnesses of the overlap-query
# fixtures (sims/triggers, sims/buttons), built with the flags, shims and
# reference library of oracle/Makefile:
#     make -C oracle -f overlap.mk overlap
include Makefile

# sims/triggers: broadphase and standalone overlap tasks only (generic harness rule)
# sims/buttons: XPBD with sphere - hull contacts, so the release-built narrowphase
# objects as for sims/balls (see Makefile)
$(OUT)/ref_buttons: harness_buttons.cpp ../sims/buttons/sim.cpp ../sims/buttons/sim.hpp harness.hpp \
                    $(BALLS_NDEBUG) $(OUT)/libmadrona_ref.a
	$(CXX) $(CXXFLAGS) -I../sims/buttons harness_buttons.cpp ../sims/buttons/sim.cpp \
	  $(BALLS_NDEBUG) $(OUT)/libmadrona_ref.a -lpthread -o $@

overlap: $(OUT)/ref_triggers $(OUT)/ref_buttons

.PHONY: overlap
