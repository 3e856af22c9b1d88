# TEST INFRASTRUCTURE ONLY -- navigation meshes on the reference CPU backend, built with the
# flags, shims and reference library of oracle/Makefile:
#     make -C oracle -f navmesh.mk navmesh
#   * ref_navmesh: the fixture sims/navmesh, with the reference's src/common/navmesh.cpp
#     compiled where it lies;
#   * navmesh_probe_ref / navmesh_probe_mine: oracle/navmesh_probe.cpp against the
#     reference's navmesh (headers + navmesh.cpp) and against the engine's device headers,
#     whose Navmesh::buildArrays is what the host builder (mb2_navmesh_create) runs.
include Makefile

navmesh: $(OUT)/ref_navmesh $(OUT)/navmesh_probe_ref $(OUT)/navmesh_probe_mine

$(OUT)/ref_common_navmesh.o: $(REF)/src/common/navmesh.cpp | $(OUT)
	$(CXX) $(CXXFLAGS) -I$(REF)/src/common -c $< -o $@

$(OUT)/ref_navmesh: harness_navmesh.cpp ../sims/navmesh/sim.cpp ../sims/navmesh/sim.hpp ../sims/navmesh/plan.hpp \
                    harness.hpp $(OUT)/ref_common_navmesh.o $(OUT)/libmadrona_ref.a
	$(CXX) $(CXXFLAGS) -I../sims/navmesh harness_navmesh.cpp ../sims/navmesh/sim.cpp \
	  $(OUT)/ref_common_navmesh.o $(OUT)/libmadrona_ref.a -lpthread -o $@

$(OUT)/navmesh_probe_ref: navmesh_probe.cpp ../sims/navmesh/plan.hpp $(OUT)/ref_common_navmesh.o \
                          $(OUT)/libmadrona_ref.a | $(OUT)
	$(CXX) $(CXXFLAGS) -DPROBE_REF navmesh_probe.cpp $(OUT)/ref_common_navmesh.o $(OUT)/libmadrona_ref.a \
	  -lpthread -o $@

$(OUT)/navmesh_probe_mine: navmesh_probe.cpp ../sims/navmesh/plan.hpp ../madrona_b200/device/madrona/navmesh.hpp \
                           ../madrona_b200/device/madrona/utils.hpp ../madrona_b200/device/madrona/memory.hpp | $(OUT)
	$(CXX) $(KATFLAGS) -I../madrona_b200/device navmesh_probe.cpp -o $@

.PHONY: navmesh
