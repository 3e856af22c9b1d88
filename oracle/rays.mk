# TEST INFRASTRUCTURE ONLY -- the reference harness of the physics ray fixture (sims/rays),
# built with the flags, shims and reference library of oracle/Makefile and, like
# oracle/crowd.mk, the reference's narrowphase and geometry built the way upstream ships them
# (-DNDEBUG).  Only the sphere-free build: the reference's traceRay asserts on spheres.
#     make -C oracle -f rays.mk rays
include Makefile

rays: $(OUT)/ref_rays

$(OUT)/ref_rays: harness_rays.cpp ../sims/rays/sim.cpp ../sims/rays/sim.hpp harness.hpp \
                 $(BALLS_NDEBUG) $(OUT)/libmadrona_ref.a
	$(CXX) $(CXXFLAGS) -I../sims/rays harness_rays.cpp ../sims/rays/sim.cpp \
	  $(BALLS_NDEBUG) $(OUT)/libmadrona_ref.a -lpthread -o $@

.PHONY: rays
