# TEST INFRASTRUCTURE ONLY -- the reference harness of the large-world fixture
# (sims/crowd), built with the flags, shims and reference library of oracle/Makefile and,
# like sims/balls and sims/hullpile (spheres against hulls), the reference's narrowphase
# and geometry built the way upstream ships them (-DNDEBUG), and the same fixture built with
# a second rigid-body archetype (-DCROWD_TWO_ARCHETYPES=1, sims/fixtures.py crowd2):
#     make -C oracle -f crowd.mk crowd
include Makefile

crowd: $(OUT)/ref_crowd $(OUT)/ref_crowd2

$(OUT)/ref_crowd: harness_crowd.cpp ../sims/crowd/sim.cpp ../sims/crowd/sim.hpp harness.hpp \
                  $(BALLS_NDEBUG) $(OUT)/libmadrona_ref.a
	$(CXX) $(CXXFLAGS) -I../sims/crowd harness_crowd.cpp ../sims/crowd/sim.cpp \
	  $(BALLS_NDEBUG) $(OUT)/libmadrona_ref.a -lpthread -o $@

$(OUT)/ref_crowd2: harness_crowd.cpp ../sims/crowd/sim.cpp ../sims/crowd/sim.hpp harness.hpp \
                   $(BALLS_NDEBUG) $(OUT)/libmadrona_ref.a
	$(CXX) $(CXXFLAGS) -DCROWD_TWO_ARCHETYPES=1 -I../sims/crowd harness_crowd.cpp ../sims/crowd/sim.cpp \
	  $(BALLS_NDEBUG) $(OUT)/libmadrona_ref.a -lpthread -o $@

.PHONY: crowd
