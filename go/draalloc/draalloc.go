// Package draalloc binds libdra_alloc.so (include/dra_alloc.h) with cgo.
//
// UNBUILT: the image this repository is developed in has no Go toolchain (`go version`: command not found),
// so this file has never been compiled.  It is the binding a maintainer of NVIDIA/k8s-dra-driver would add
// next to cmd/nvidia-dra-controller to put the H100 allocation path behind the classic
// controller.Driver surface (Allocate / UnsuitableNodes / Deallocate).  The C++ layer in
// k8s-dra-driver_b200/csrc/dra_host.cpp is the same logic, built and tested (tests/cpp/driver_test.cpp).
package draalloc

/*
#cgo CFLAGS: -I${SRCDIR}/../../include
#cgo LDFLAGS: -L${SRCDIR}/../../k8s-dra-driver_b200 -ldra_alloc
#include <stdlib.h>
#include "dra_alloc.h"
*/
import "C"

import (
	"errors"
	"fmt"
	"runtime"
	"sync"
	"unsafe"
)

// Records: identical layout to the C structs (spec/ALLOCATION.md §1).
type GpuRec struct {
	Busy       uint16
	Flags      uint8
	Model      uint8
	MemFreeMiB uint32
	Node       uint32
	ShareCnt   uint16
	_          uint16
}

type ClaimRec struct {
	Kind        uint8
	Profile     uint8
	Count       uint16
	Node        uint32
	MemLimitMiB uint32
	Group       uint32
}

type OutRec struct {
	Gpu     uint32
	Start   uint8
	Size    uint8
	Profile uint8
	Status  uint8
}

const (
	KindGpu    = 0
	KindMig    = 1
	KindShared = 2

	GpuMigEnabled    = 0x01
	GpuFullAllocated = 0x02
	GpuUnavailable   = 0x04

	StOK          = 0
	StPod         = 6 // pod mode: the pod does not fit on the node
	StSearchLimit = 7

	FlagExhaustive = 0x4 // DRA_F_EXHAUSTIVE: backtracking placement search (spec §12)
	CfgResident    = 0x8 // DRA_CFG_RESIDENT: resident kernel + doorbell for small batches
)

// Context owns one dra_ctx (one CUDA device, one stream, one inventory).  Calls are serialised, as the
// reference serialises its own (cmd/nvidia-dra-plugin/driver.go:119-120).
type Context struct {
	mu sync.Mutex
	h  *C.dra_ctx
}

func lastError(h *C.dra_ctx) error { return errors.New(C.GoString(C.dra_last_error(h))) }

func NewContext(device int, cfgFlags uint32) (*Context, error) {
	cfg := C.dra_cfg{abi_version: C.DRA_ABI_VERSION, device: C.int32_t(device), flags: C.uint32_t(cfgFlags)}
	var h *C.dra_ctx
	if rc := C.dra_ctx_create(&cfg, &h); rc != 0 {
		return nil, fmt.Errorf("dra_ctx_create: %w", lastError(nil))
	}
	c := &Context{h: h}
	runtime.SetFinalizer(c, func(c *Context) { c.Close() })
	return c, nil
}

func (c *Context) Close() {
	c.mu.Lock()
	defer c.mu.Unlock()
	if c.h != nil {
		C.dra_ctx_destroy(c.h)
		c.h = nil
	}
}

// SetPlacementTable mirrors what deviceLib.getGpuInfo collects per GPU model (nvlib.go:244-295).
func (c *Context) SetPlacementTable(model uint32, sizes [16]uint8, startMasks [16]uint16) error {
	var t C.dra_profile_tbl
	for p := 0; p < 16; p++ {
		t.ent[p].size = C.uint8_t(sizes[p])
		t.ent[p].start_mask = C.uint16_t(startMasks[p])
	}
	c.mu.Lock()
	defer c.mu.Unlock()
	if rc := C.dra_set_placement_table(c.h, C.uint32_t(model), &t); rc != 0 {
		return lastError(c.h)
	}
	return nil
}

func (c *Context) SetInventory(gpus []GpuRec, nodeOff []uint32) error {
	c.mu.Lock()
	defer c.mu.Unlock()
	var gp *C.dra_gpu_rec
	if len(gpus) > 0 {
		gp = (*C.dra_gpu_rec)(unsafe.Pointer(&gpus[0]))
	}
	rc := C.dra_set_inventory(c.h, gp, C.uint32_t(len(gpus)),
		(*C.uint32_t)(unsafe.Pointer(&nodeOff[0])), C.uint32_t(len(nodeOff)-1))
	if rc != 0 {
		return lastError(c.h)
	}
	return nil
}

// AllocateBatch = controller.Driver.Allocate batched over pods: every claim carries its selectedNode.
// outOff may be nil when every claim wants exactly one device.  cgo blocks the calling OS thread for the
// duration of the call (tens of microseconds per 10k claims), so keep calls batch-sized.
func (c *Context) AllocateBatch(claims []ClaimRec, outOff []uint32, nOut int) ([]OutRec, error) {
	out := make([]OutRec, nOut)
	if len(claims) == 0 {
		return out, nil
	}
	var oo *C.uint32_t
	if outOff != nil {
		oo = (*C.uint32_t)(unsafe.Pointer(&outOff[0]))
	}
	c.mu.Lock()
	defer c.mu.Unlock()
	rc := C.dra_allocate_batch(c.h, (*C.dra_claim_rec)(unsafe.Pointer(&claims[0])), C.uint32_t(len(claims)),
		oo, (*C.dra_out_rec)(unsafe.Pointer(&out[0])), C.uint32_t(nOut), 0)
	if rc != 0 {
		return nil, lastError(c.h)
	}
	return out, nil
}

// UnsuitableBatch = controller.Driver.UnsuitableNodes batched over pods; bit k of the result is set when
// the k-th (pod, candidate node) pair is suitable.
func (c *Context) UnsuitableBatch(claims []ClaimRec, podOff, candNodes, candOff []uint32, flags uint32) ([]byte, error) {
	nPod := len(podOff) - 1
	bits := make([]byte, (int(candOff[nPod])+7)/8+1)
	c.mu.Lock()
	defer c.mu.Unlock()
	var cp *C.dra_claim_rec
	if len(claims) > 0 {
		cp = (*C.dra_claim_rec)(unsafe.Pointer(&claims[0]))
	}
	var cn *C.uint32_t
	if len(candNodes) > 0 {
		cn = (*C.uint32_t)(unsafe.Pointer(&candNodes[0]))
	}
	rc := C.dra_unsuitable_batch(c.h, cp, C.uint32_t(len(claims)),
		(*C.uint32_t)(unsafe.Pointer(&podOff[0])), C.uint32_t(nPod), cn,
		(*C.uint32_t)(unsafe.Pointer(&candOff[0])), (*C.uint8_t)(unsafe.Pointer(&bits[0])), C.uint32_t(flags))
	if rc != 0 {
		return nil, lastError(c.h)
	}
	return bits, nil
}

// AllocatePodsBatch = Allocate with pod boundaries (spec §12): every pod (claims podOff[p]..podOff[p+1], one node)
// is placed atomically; with FlagExhaustive its MIG claims are placed by the backtracking search over every valid
// placement — what the classic mig.allocate did after UnsuitableNodes had found an assignment.
func (c *Context) AllocatePodsBatch(claims []ClaimRec, podOff, outOff []uint32, nOut int, flags uint32) ([]OutRec, error) {
	out := make([]OutRec, nOut)
	if len(claims) == 0 {
		return out, nil
	}
	var oo *C.uint32_t
	if outOff != nil {
		oo = (*C.uint32_t)(unsafe.Pointer(&outOff[0]))
	}
	c.mu.Lock()
	defer c.mu.Unlock()
	rc := C.dra_allocate_pods_batch(c.h, (*C.dra_claim_rec)(unsafe.Pointer(&claims[0])), C.uint32_t(len(claims)),
		(*C.uint32_t)(unsafe.Pointer(&podOff[0])), C.uint32_t(len(podOff)-1),
		oo, (*C.dra_out_rec)(unsafe.Pointer(&out[0])), C.uint32_t(nOut), C.uint32_t(flags))
	if rc != 0 {
		return nil, lastError(c.h)
	}
	return out, nil
}

// PlacePodsBatch chooses the node and allocates in one call (dra_place_pods_batch, spec §13): pods in input order, each on
// the first of its candidates cands[candOff[p]:candOff[p+1]] where all its claims fit given what the pods before it took.
// cands == candOff == nil: every node, ascending.  The claims' node fields are ignored.  Returns the OutRecs and, per pod,
// the node it was placed on (0xFFFFFFFF: none).  nOut counts slots as if every claim named a node.  Unbuilt, like the rest
// of this file.
func (c *Context) PlacePodsBatch(claims []ClaimRec, podOff []uint32, cands, candOff []uint32, outOff []uint32, nOut int,
	flags uint32) ([]OutRec, []uint32, error) {
	out := make([]OutRec, nOut)
	podNode := make([]uint32, len(podOff)-1)
	if len(podNode) == 0 {
		return out, podNode, nil
	}
	var cp *C.dra_claim_rec
	var oo, cn, co *C.uint32_t
	if len(claims) > 0 {
		cp = (*C.dra_claim_rec)(unsafe.Pointer(&claims[0]))
	}
	if outOff != nil {
		oo = (*C.uint32_t)(unsafe.Pointer(&outOff[0]))
	}
	if candOff != nil {
		co = (*C.uint32_t)(unsafe.Pointer(&candOff[0]))
		if len(cands) == 0 {
			cands = []uint32{0} // an empty list still needs an address (nil means the dense form)
		}
		cn = (*C.uint32_t)(unsafe.Pointer(&cands[0]))
	}
	var op *C.dra_out_rec
	if nOut > 0 {
		op = (*C.dra_out_rec)(unsafe.Pointer(&out[0]))
	}
	c.mu.Lock()
	defer c.mu.Unlock()
	rc := C.dra_place_pods_batch(c.h, cp, C.uint32_t(len(claims)), (*C.uint32_t)(unsafe.Pointer(&podOff[0])),
		C.uint32_t(len(podNode)), cn, co, oo, op, C.uint32_t(nOut), (*C.uint32_t)(unsafe.Pointer(&podNode[0])), C.uint32_t(flags))
	if rc != 0 {
		return nil, nil, lastError(c.h)
	}
	return out, podNode, nil
}

// Running pods for PreemptBatch: the arrays DeallocateBatch takes for their allocations (outOff nil: slot i), split into
// pods by PodOff, one priority per pod.  Pod index order is start order, earliest first.
type RunningPods struct {
	Claims []ClaimRec
	PodOff []uint32
	Prio   []int32
	OutOff []uint32
	Out    []OutRec
}

// Preemption answer (spec §14).  Per pair: Status (DRA_PRE_*) and, for EVICT, the victim count.  Per pod: the node to
// evict on (0xFFFFFFFF: none), its status, the full victim count and the first maxVictims victims as running-pod indices
// (row p at Victims[p*maxVictims:], padded with 0xFFFFFFFF).
type Preemption struct {
	PairStatus  []uint8
	PairVictims []uint32
	PodNode     []uint32
	PodStatus   []uint8
	NVictims    []uint32
	Victims     []uint32
}

// PreemptBatch answers kube-scheduler's PostFilter for pods whose GPU claims fit nowhere (dra_preempt_batch, spec §14):
// per candidate node the lower-priority running pods to evict, and per pod the node to evict them on.  Pure: the
// inventory is not written.  cands == candOff == nil: every node, ascending (nNode: the inventory's node count, which
// sizes the per-pair outputs of that form).  Unbuilt, like the rest of this file.
func (c *Context) PreemptBatch(claims []ClaimRec, podOff []uint32, prio []int32, cands, candOff []uint32, nNode int,
	run RunningPods, maxVictims int, flags uint32) (*Preemption, error) {
	nPod := len(podOff) - 1
	if nPod <= 0 || len(run.PodOff) == 0 {
		return &Preemption{}, nil
	}
	nPair := nPod * nNode
	var cn, co *C.uint32_t
	if candOff != nil {
		nPair = int(candOff[nPod])
		co = (*C.uint32_t)(unsafe.Pointer(&candOff[0]))
		if len(cands) == 0 {
			cands = []uint32{0} // an empty list still needs an address (nil means the dense form)
		}
		cn = (*C.uint32_t)(unsafe.Pointer(&cands[0]))
	}
	r := &Preemption{make([]uint8, nPair+1), make([]uint32, nPair+1), make([]uint32, nPod), make([]uint8, nPod),
		make([]uint32, nPod), make([]uint32, nPod*maxVictims+1)}
	var cp, rcp *C.dra_claim_rec
	if len(claims) > 0 {
		cp = (*C.dra_claim_rec)(unsafe.Pointer(&claims[0]))
	}
	if len(run.Claims) > 0 {
		rcp = (*C.dra_claim_rec)(unsafe.Pointer(&run.Claims[0]))
	}
	var rp *C.int32_t
	if len(run.Prio) > 0 {
		rp = (*C.int32_t)(unsafe.Pointer(&run.Prio[0]))
	}
	var roo *C.uint32_t
	if run.OutOff != nil {
		roo = (*C.uint32_t)(unsafe.Pointer(&run.OutOff[0]))
	}
	var rop *C.dra_out_rec
	if len(run.Out) > 0 {
		rop = (*C.dra_out_rec)(unsafe.Pointer(&run.Out[0]))
	}
	// the struct handed to C holds Go pointers: cgo accepts that only for pinned memory
	var pin runtime.Pinner
	defer pin.Unpin()
	for _, q := range []unsafe.Pointer{unsafe.Pointer(rcp), unsafe.Pointer(&run.PodOff[0]), unsafe.Pointer(rp),
		unsafe.Pointer(roo), unsafe.Pointer(rop)} {
		if q != nil {
			pin.Pin(q)
		}
	}
	cr := C.dra_running_pods{claims: rcp, n_claim: C.uint32_t(len(run.Claims)),
		pod_off: (*C.uint32_t)(unsafe.Pointer(&run.PodOff[0])), n_pod: C.uint32_t(len(run.PodOff) - 1), prio: rp,
		out_off: roo, out: rop, n_out: C.uint32_t(len(run.Out))}
	var vp *C.uint32_t
	if maxVictims > 0 {
		vp = (*C.uint32_t)(unsafe.Pointer(&r.Victims[0]))
	}
	c.mu.Lock()
	defer c.mu.Unlock()
	rc := C.dra_preempt_batch(c.h, cp, C.uint32_t(len(claims)), (*C.uint32_t)(unsafe.Pointer(&podOff[0])),
		(*C.int32_t)(unsafe.Pointer(&prio[0])), C.uint32_t(nPod), cn, co, &cr,
		(*C.uint8_t)(unsafe.Pointer(&r.PairStatus[0])), (*C.uint32_t)(unsafe.Pointer(&r.PairVictims[0])),
		(*C.uint32_t)(unsafe.Pointer(&r.PodNode[0])), (*C.uint8_t)(unsafe.Pointer(&r.PodStatus[0])),
		(*C.uint32_t)(unsafe.Pointer(&r.NVictims[0])), vp, C.uint32_t(maxVictims), C.uint32_t(flags))
	if rc != 0 {
		return nil, lastError(c.h)
	}
	r.PairStatus, r.PairVictims, r.Victims = r.PairStatus[:nPair], r.PairVictims[:nPair], r.Victims[:nPod*maxVictims]
	return r, nil
}

// PdbNone: a running pod that counts against no disruption budget.
const PdbNone = 0xFFFFFFFF

// DisruptionBudgets for PreemptPdbBatch (spec §14, "Disruption budgets"): RunPdb[r] the budget running pod r counts
// against (PdbNone for none, also for a pod in its budget's DisruptedPods), Allowed[b] each budget's
// status.disruptionsAllowed.  Both empty: no budgets.
type DisruptionBudgets struct {
	RunPdb  []uint32
	Allowed []int32
}

// Preemption answer with disruption budgets: Preemption, plus per pair the violating victims of an EVICT pair and per
// pod the chosen pair's.
type PreemptionPdb struct {
	Preemption
	PairViolations []uint32
	PodViolations  []uint32
}

// PreemptPdbBatch is PreemptBatch honouring PodDisruptionBudgets (dra_preempt_pdb_batch): on each candidate node the
// running pods whose eviction would violate their budget are reprieved first, and a pod's node is the one with the fewest
// violating victims before any other criterion.  Unbuilt, like the rest of this file.
func (c *Context) PreemptPdbBatch(claims []ClaimRec, podOff []uint32, prio []int32, cands, candOff []uint32, nNode int,
	run RunningPods, budgets DisruptionBudgets, maxVictims int, flags uint32) (*PreemptionPdb, error) {
	nPod := len(podOff) - 1
	if nPod <= 0 || len(run.PodOff) == 0 {
		return &PreemptionPdb{}, nil
	}
	nPair := nPod * nNode
	var cn, co *C.uint32_t
	if candOff != nil {
		nPair = int(candOff[nPod])
		co = (*C.uint32_t)(unsafe.Pointer(&candOff[0]))
		if len(cands) == 0 {
			cands = []uint32{0} // an empty list still needs an address (nil means the dense form)
		}
		cn = (*C.uint32_t)(unsafe.Pointer(&cands[0]))
	}
	r := &PreemptionPdb{Preemption{make([]uint8, nPair+1), make([]uint32, nPair+1), make([]uint32, nPod),
		make([]uint8, nPod), make([]uint32, nPod), make([]uint32, nPod*maxVictims+1)},
		make([]uint32, nPair+1), make([]uint32, nPod)}
	var cp, rcp *C.dra_claim_rec
	if len(claims) > 0 {
		cp = (*C.dra_claim_rec)(unsafe.Pointer(&claims[0]))
	}
	if len(run.Claims) > 0 {
		rcp = (*C.dra_claim_rec)(unsafe.Pointer(&run.Claims[0]))
	}
	var rp *C.int32_t
	if len(run.Prio) > 0 {
		rp = (*C.int32_t)(unsafe.Pointer(&run.Prio[0]))
	}
	var roo *C.uint32_t
	if run.OutOff != nil {
		roo = (*C.uint32_t)(unsafe.Pointer(&run.OutOff[0]))
	}
	var rop *C.dra_out_rec
	if len(run.Out) > 0 {
		rop = (*C.dra_out_rec)(unsafe.Pointer(&run.Out[0]))
	}
	var bpdb *C.uint32_t
	if len(budgets.RunPdb) > 0 {
		bpdb = (*C.uint32_t)(unsafe.Pointer(&budgets.RunPdb[0]))
	}
	var bal *C.int32_t
	if len(budgets.Allowed) > 0 {
		bal = (*C.int32_t)(unsafe.Pointer(&budgets.Allowed[0]))
	}
	// the structs handed to C hold Go pointers: cgo accepts that only for pinned memory
	var pin runtime.Pinner
	defer pin.Unpin()
	for _, q := range []unsafe.Pointer{unsafe.Pointer(rcp), unsafe.Pointer(&run.PodOff[0]), unsafe.Pointer(rp),
		unsafe.Pointer(roo), unsafe.Pointer(rop), unsafe.Pointer(bpdb), unsafe.Pointer(bal)} {
		if q != nil {
			pin.Pin(q)
		}
	}
	cr := C.dra_running_pods{claims: rcp, n_claim: C.uint32_t(len(run.Claims)),
		pod_off: (*C.uint32_t)(unsafe.Pointer(&run.PodOff[0])), n_pod: C.uint32_t(len(run.PodOff) - 1), prio: rp,
		out_off: roo, out: rop, n_out: C.uint32_t(len(run.Out))}
	cb := C.dra_disruption_budgets{run_pdb: bpdb, allowed: bal, n_pdb: C.uint32_t(len(budgets.Allowed))}
	var vp *C.uint32_t
	if maxVictims > 0 {
		vp = (*C.uint32_t)(unsafe.Pointer(&r.Victims[0]))
	}
	c.mu.Lock()
	defer c.mu.Unlock()
	rc := C.dra_preempt_pdb_batch(c.h, cp, C.uint32_t(len(claims)), (*C.uint32_t)(unsafe.Pointer(&podOff[0])),
		(*C.int32_t)(unsafe.Pointer(&prio[0])), C.uint32_t(nPod), cn, co, &cr, &cb,
		(*C.uint8_t)(unsafe.Pointer(&r.PairStatus[0])), (*C.uint32_t)(unsafe.Pointer(&r.PairVictims[0])),
		(*C.uint32_t)(unsafe.Pointer(&r.PairViolations[0])), (*C.uint32_t)(unsafe.Pointer(&r.PodNode[0])),
		(*C.uint8_t)(unsafe.Pointer(&r.PodStatus[0])), (*C.uint32_t)(unsafe.Pointer(&r.NVictims[0])),
		(*C.uint32_t)(unsafe.Pointer(&r.PodViolations[0])), vp, C.uint32_t(maxVictims), C.uint32_t(flags))
	if rc != 0 {
		return nil, lastError(c.h)
	}
	r.PairStatus, r.PairVictims, r.Victims = r.PairStatus[:nPair], r.PairVictims[:nPair], r.Victims[:nPod*maxVictims]
	r.PairViolations = r.PairViolations[:nPair]
	return r, nil
}

// Preempt-and-place answer (spec §15).  Per pod: the node chosen (0xFFFFFFFF: none) and its status (DRA_PRE_*).  Per
// running pod: the pending pod that evicted it, 0xFFFFFFFF when none.
type PreemptPlacement struct {
	Out       []OutRec
	PodNode   []uint32
	PodStatus []uint8
	EvictedBy []uint32
}

// PreemptPlaceBatch runs PostFilter and Reserve for a whole batch in one call (dra_preempt_place_batch, spec §15): pods
// in input order, each judged as PreemptBatch judges it on the inventory the pods before it left, then applied — its
// victims released, the pod allocated on the chosen node.  Candidates as PlaceBatch (cands == candOff == nil: every
// node, ascending); outOff / nOut as PlaceBatch.  The call releases the victims itself: do not pass them to
// DeallocateBatch again.  Unbuilt, like the rest of this file.
func (c *Context) PreemptPlaceBatch(claims []ClaimRec, podOff []uint32, prio []int32, cands, candOff []uint32,
	run RunningPods, outOff []uint32, nOut int, flags uint32) (*PreemptPlacement, error) {
	nPod := len(podOff) - 1
	if nPod <= 0 || len(run.PodOff) == 0 {
		return &PreemptPlacement{Out: make([]OutRec, nOut)}, nil
	}
	r := &PreemptPlacement{make([]OutRec, nOut+1), make([]uint32, nPod), make([]uint8, nPod), make([]uint32, len(run.PodOff))}
	var cp, rcp *C.dra_claim_rec
	var oo, cn, co, roo *C.uint32_t
	if len(claims) > 0 {
		cp = (*C.dra_claim_rec)(unsafe.Pointer(&claims[0]))
	}
	if outOff != nil {
		oo = (*C.uint32_t)(unsafe.Pointer(&outOff[0]))
	}
	if candOff != nil {
		co = (*C.uint32_t)(unsafe.Pointer(&candOff[0]))
		if len(cands) == 0 {
			cands = []uint32{0} // an empty list still needs an address (nil means the dense form)
		}
		cn = (*C.uint32_t)(unsafe.Pointer(&cands[0]))
	}
	if len(run.Claims) > 0 {
		rcp = (*C.dra_claim_rec)(unsafe.Pointer(&run.Claims[0]))
	}
	var rp *C.int32_t
	if len(run.Prio) > 0 {
		rp = (*C.int32_t)(unsafe.Pointer(&run.Prio[0]))
	}
	if run.OutOff != nil {
		roo = (*C.uint32_t)(unsafe.Pointer(&run.OutOff[0]))
	}
	var rop *C.dra_out_rec
	if len(run.Out) > 0 {
		rop = (*C.dra_out_rec)(unsafe.Pointer(&run.Out[0]))
	}
	// the struct handed to C holds Go pointers: cgo accepts that only for pinned memory
	var pin runtime.Pinner
	defer pin.Unpin()
	for _, q := range []unsafe.Pointer{unsafe.Pointer(rcp), unsafe.Pointer(&run.PodOff[0]), unsafe.Pointer(rp),
		unsafe.Pointer(roo), unsafe.Pointer(rop)} {
		if q != nil {
			pin.Pin(q)
		}
	}
	cr := C.dra_running_pods{claims: rcp, n_claim: C.uint32_t(len(run.Claims)),
		pod_off: (*C.uint32_t)(unsafe.Pointer(&run.PodOff[0])), n_pod: C.uint32_t(len(run.PodOff) - 1), prio: rp,
		out_off: roo, out: rop, n_out: C.uint32_t(len(run.Out))}
	c.mu.Lock()
	defer c.mu.Unlock()
	rc := C.dra_preempt_place_batch(c.h, cp, C.uint32_t(len(claims)), (*C.uint32_t)(unsafe.Pointer(&podOff[0])),
		(*C.int32_t)(unsafe.Pointer(&prio[0])), C.uint32_t(nPod), cn, co, &cr, oo,
		(*C.dra_out_rec)(unsafe.Pointer(&r.Out[0])), C.uint32_t(nOut), (*C.uint32_t)(unsafe.Pointer(&r.PodNode[0])),
		(*C.uint8_t)(unsafe.Pointer(&r.PodStatus[0])), (*C.uint32_t)(unsafe.Pointer(&r.EvictedBy[0])), C.uint32_t(flags))
	if rc != 0 {
		return nil, lastError(c.h)
	}
	r.Out, r.EvictedBy = r.Out[:nOut], r.EvictedBy[:len(run.PodOff)-1]
	return r, nil
}

// cRunning: run as dra_running_pods.  The struct holds Go pointers, which cgo accepts only for pinned memory: pin keeps
// them pinned until the caller unpins it.
func cRunning(run RunningPods, pin *runtime.Pinner) C.dra_running_pods {
	var rcp *C.dra_claim_rec
	var rp *C.int32_t
	var roo *C.uint32_t
	var rop *C.dra_out_rec
	if len(run.Claims) > 0 {
		rcp = (*C.dra_claim_rec)(unsafe.Pointer(&run.Claims[0]))
	}
	if len(run.Prio) > 0 {
		rp = (*C.int32_t)(unsafe.Pointer(&run.Prio[0]))
	}
	if run.OutOff != nil {
		roo = (*C.uint32_t)(unsafe.Pointer(&run.OutOff[0]))
	}
	if len(run.Out) > 0 {
		rop = (*C.dra_out_rec)(unsafe.Pointer(&run.Out[0]))
	}
	for _, q := range []unsafe.Pointer{unsafe.Pointer(rcp), unsafe.Pointer(&run.PodOff[0]), unsafe.Pointer(rp),
		unsafe.Pointer(roo), unsafe.Pointer(rop)} {
		if q != nil {
			pin.Pin(q)
		}
	}
	return C.dra_running_pods{claims: rcp, n_claim: C.uint32_t(len(run.Claims)),
		pod_off: (*C.uint32_t)(unsafe.Pointer(&run.PodOff[0])), n_pod: C.uint32_t(len(run.PodOff) - 1), prio: rp,
		out_off: roo, out: rop, n_out: C.uint32_t(len(run.Out))}
}

// PreemptWhyBatch says why preemption judged each candidate node as it did (dra_preempt_why_batch, spec §19): per pair the
// status PreemptBatch gives it (pairStatus, may be nil), a reason and a blocking claim, and the per-pod and per-claim
// tallies (podWhy, claimBlocks, may be nil), laid out as UnsuitableWhyBatch's.  Every slice is the caller's, sized as
// the C call documents (pairWhy and pairClaim: one entry per pair).  Pure.  Unbuilt, like the rest of this file.
func (c *Context) PreemptWhyBatch(claims []ClaimRec, podOff []uint32, prio []int32, cands, candOff []uint32, run RunningPods,
	pairStatus, pairWhy []uint8, pairClaim, podWhy, claimBlocks []uint32, flags uint32) error {
	nPod := len(podOff) - 1
	if nPod <= 0 || len(run.PodOff) == 0 {
		return nil
	}
	var cp *C.dra_claim_rec
	var cn, co *C.uint32_t
	if len(claims) > 0 {
		cp = (*C.dra_claim_rec)(unsafe.Pointer(&claims[0]))
	}
	if candOff != nil {
		co = (*C.uint32_t)(unsafe.Pointer(&candOff[0]))
		if len(cands) == 0 {
			cands = []uint32{0} // an empty list still needs an address (nil means the dense form)
		}
		cn = (*C.uint32_t)(unsafe.Pointer(&cands[0]))
	}
	var pin runtime.Pinner
	defer pin.Unpin()
	cr := cRunning(run, &pin)
	c.mu.Lock()
	defer c.mu.Unlock()
	rc := C.dra_preempt_why_batch(c.h, cp, C.uint32_t(len(claims)), (*C.uint32_t)(unsafe.Pointer(&podOff[0])),
		(*C.int32_t)(unsafe.Pointer(&prio[0])), C.uint32_t(nPod), cn, co, &cr, (*C.uint8_t)(sliceAddr8(pairStatus)),
		(*C.uint8_t)(sliceAddr8(pairWhy)), (*C.uint32_t)(sliceAddr32(pairClaim)), (*C.uint32_t)(sliceAddr32(podWhy)),
		(*C.uint32_t)(sliceAddr32(claimBlocks)), C.uint32_t(flags))
	if rc != 0 {
		return lastError(c.h)
	}
	return nil
}

// PreemptPlaceWhyBatch is PreemptPlaceBatch that also says why each pod was judged as it was on each candidate
// (dra_preempt_place_why_batch, spec §19): the reason outputs of PreemptWhyBatch, each pair judged on the state its pod
// met.  Placement, eviction and the inventory are PreemptPlaceBatch's.  Unbuilt, like the rest of this file.
func (c *Context) PreemptPlaceWhyBatch(claims []ClaimRec, podOff []uint32, prio []int32, cands, candOff []uint32,
	run RunningPods, outOff []uint32, nOut int, pairStatus, pairWhy []uint8, pairClaim, podWhy, claimBlocks []uint32,
	flags uint32) (*PreemptPlacement, error) {
	nPod := len(podOff) - 1
	if nPod <= 0 || len(run.PodOff) == 0 {
		return &PreemptPlacement{Out: make([]OutRec, nOut)}, nil
	}
	r := &PreemptPlacement{make([]OutRec, nOut+1), make([]uint32, nPod), make([]uint8, nPod), make([]uint32, len(run.PodOff))}
	var cp *C.dra_claim_rec
	var oo, cn, co *C.uint32_t
	if len(claims) > 0 {
		cp = (*C.dra_claim_rec)(unsafe.Pointer(&claims[0]))
	}
	if outOff != nil {
		oo = (*C.uint32_t)(unsafe.Pointer(&outOff[0]))
	}
	if candOff != nil {
		co = (*C.uint32_t)(unsafe.Pointer(&candOff[0]))
		if len(cands) == 0 {
			cands = []uint32{0} // an empty list still needs an address (nil means the dense form)
		}
		cn = (*C.uint32_t)(unsafe.Pointer(&cands[0]))
	}
	var pin runtime.Pinner
	defer pin.Unpin()
	cr := cRunning(run, &pin)
	c.mu.Lock()
	defer c.mu.Unlock()
	rc := C.dra_preempt_place_why_batch(c.h, cp, C.uint32_t(len(claims)), (*C.uint32_t)(unsafe.Pointer(&podOff[0])),
		(*C.int32_t)(unsafe.Pointer(&prio[0])), C.uint32_t(nPod), cn, co, &cr, oo,
		(*C.dra_out_rec)(unsafe.Pointer(&r.Out[0])), C.uint32_t(nOut), (*C.uint32_t)(unsafe.Pointer(&r.PodNode[0])),
		(*C.uint8_t)(unsafe.Pointer(&r.PodStatus[0])), (*C.uint32_t)(unsafe.Pointer(&r.EvictedBy[0])),
		(*C.uint8_t)(sliceAddr8(pairStatus)), (*C.uint8_t)(sliceAddr8(pairWhy)), (*C.uint32_t)(sliceAddr32(pairClaim)),
		(*C.uint32_t)(sliceAddr32(podWhy)), (*C.uint32_t)(sliceAddr32(claimBlocks)), C.uint32_t(flags))
	if rc != 0 {
		return nil, lastError(c.h)
	}
	r.Out, r.EvictedBy = r.Out[:nOut], r.EvictedBy[:len(run.PodOff)-1]
	return r, nil
}

// sliceAddr8 / sliceAddr32: the first element's address, nil for an empty or nil slice (an optional output)
func sliceAddr8(b []uint8) unsafe.Pointer {
	if len(b) == 0 {
		return nil
	}
	return unsafe.Pointer(&b[0])
}

func sliceAddr32(b []uint32) unsafe.Pointer {
	if len(b) == 0 {
		return nil
	}
	return unsafe.Pointer(&b[0])
}

// Pod-capacity answer (spec §16).  Per pair (candOff order; dense: pod*nNode + node): the copies of the pod the node
// still takes and why counting stopped (DRA_ST_OK: maxCopies reached, DRA_ST_POD, DRA_ST_SEARCH_LIMIT, DRA_ST_INVALID).
// Per pod: the sum over its pairs and how many of them take at least one copy.
type PodCapacity struct {
	PairCopies []uint16
	PairStop   []uint8
	PodTotal   []uint64
	PodNodes   []uint32
}

// PodCapacityBatch counts, for each pod and each of its candidate nodes, how many copies of the pod the node still takes,
// placed as AllocatePodsBatch would place them with the same flags, at most maxCopies (1 .. 65535) per node
// (dra_pod_capacity_batch, spec §16).  Pure.  Candidates as PlaceBatch (cands == candOff == nil: every node, ascending,
// nNode of them).  Unbuilt, like the rest of this file.
func (c *Context) PodCapacityBatch(claims []ClaimRec, podOff []uint32, cands, candOff []uint32, nNode int,
	maxCopies uint32, flags uint32) (*PodCapacity, error) {
	nPod := len(podOff) - 1
	if nPod <= 0 {
		return &PodCapacity{}, nil
	}
	nPair := nPod * nNode
	var cp *C.dra_claim_rec
	var cn, co *C.uint32_t
	if len(claims) > 0 {
		cp = (*C.dra_claim_rec)(unsafe.Pointer(&claims[0]))
	}
	if candOff != nil {
		nPair = int(candOff[nPod])
		co = (*C.uint32_t)(unsafe.Pointer(&candOff[0]))
		if len(cands) == 0 {
			cands = []uint32{0} // an empty list still needs an address (nil means the dense form)
		}
		cn = (*C.uint32_t)(unsafe.Pointer(&cands[0]))
	}
	r := &PodCapacity{make([]uint16, nPair+1), make([]uint8, nPair+1), make([]uint64, nPod), make([]uint32, nPod)}
	c.mu.Lock()
	defer c.mu.Unlock()
	rc := C.dra_pod_capacity_batch(c.h, cp, C.uint32_t(len(claims)), (*C.uint32_t)(unsafe.Pointer(&podOff[0])),
		C.uint32_t(nPod), cn, co, C.uint32_t(maxCopies), (*C.uint16_t)(unsafe.Pointer(&r.PairCopies[0])),
		(*C.uint8_t)(unsafe.Pointer(&r.PairStop[0])), (*C.uint64_t)(unsafe.Pointer(&r.PodTotal[0])),
		(*C.uint32_t)(unsafe.Pointer(&r.PodNodes[0])), C.uint32_t(flags))
	if rc != 0 {
		return nil, lastError(c.h)
	}
	r.PairCopies, r.PairStop = r.PairCopies[:nPair], r.PairStop[:nPair]
	return r, nil
}

// UnsuitableWhy is UnsuitableWhyBatch's answer (spec §17): per (pod, candidate) pair the reason (DRA_ST_*, or
// DRA_WHY_NO_NODE = 8) and the blocking claim (an index into the claims passed, or DRA_WHY_CLAIM_NONE); per pod the
// pairs of each reason (PodWhy[p*9+r]); per claim the pairs it blocks.
type UnsuitableWhy struct {
	PairWhy     []uint8
	PairClaim   []uint32
	PodWhy      []uint32
	ClaimBlocks []uint32
}

// UnsuitableWhyBatch answers UnsuitableBatch's pairs with the reason each node is unsuitable and the claim that blocks
// it (dra_unsuitable_why_batch, spec §17).  Pure.  Candidates as PlaceBatch (cands == candOff == nil: every node,
// ascending, nNode of them).  The claim indices refer to the lowered claims, in lowering order.  Unbuilt, like the rest
// of this file.
func (c *Context) UnsuitableWhyBatch(claims []ClaimRec, podOff []uint32, cands, candOff []uint32, nNode int,
	flags uint32) (*UnsuitableWhy, error) {
	nPod := len(podOff) - 1
	if nPod <= 0 {
		return &UnsuitableWhy{}, nil
	}
	nPair := nPod * nNode
	var cp *C.dra_claim_rec
	var cn, co *C.uint32_t
	if len(claims) > 0 {
		cp = (*C.dra_claim_rec)(unsafe.Pointer(&claims[0]))
	}
	if candOff != nil {
		nPair = int(candOff[nPod])
		co = (*C.uint32_t)(unsafe.Pointer(&candOff[0]))
		if len(cands) == 0 {
			cands = []uint32{0} // an empty list still needs an address (nil means the dense form)
		}
		cn = (*C.uint32_t)(unsafe.Pointer(&cands[0]))
	}
	r := &UnsuitableWhy{make([]uint8, nPair+1), make([]uint32, nPair+1), make([]uint32, nPod*9), make([]uint32, len(claims)+1)}
	c.mu.Lock()
	defer c.mu.Unlock()
	rc := C.dra_unsuitable_why_batch(c.h, cp, C.uint32_t(len(claims)), (*C.uint32_t)(unsafe.Pointer(&podOff[0])),
		C.uint32_t(nPod), cn, co, (*C.uint8_t)(unsafe.Pointer(&r.PairWhy[0])), (*C.uint32_t)(unsafe.Pointer(&r.PairClaim[0])),
		(*C.uint32_t)(unsafe.Pointer(&r.PodWhy[0])), (*C.uint32_t)(unsafe.Pointer(&r.ClaimBlocks[0])), C.uint32_t(flags))
	if rc != 0 {
		return nil, lastError(c.h)
	}
	r.PairWhy, r.PairClaim, r.ClaimBlocks = r.PairWhy[:nPair], r.PairClaim[:nPair], r.ClaimBlocks[:len(claims)]
	return r, nil
}

func (c *Context) DeallocateBatch(claims []ClaimRec, outOff []uint32, out []OutRec) error {
	if len(claims) == 0 {
		return nil
	}
	var oo *C.uint32_t
	if outOff != nil {
		oo = (*C.uint32_t)(unsafe.Pointer(&outOff[0]))
	}
	c.mu.Lock()
	defer c.mu.Unlock()
	rc := C.dra_deallocate_batch(c.h, (*C.dra_claim_rec)(unsafe.Pointer(&claims[0])), C.uint32_t(len(claims)),
		oo, (*C.dra_out_rec)(unsafe.Pointer(&out[0])), C.uint32_t(len(out)))
	if rc != 0 {
		return lastError(c.h)
	}
	return nil
}

// ---- one global batch over the GPUs of a box (one Context per GPU of ONE process) --------------------------------------
// Set-up once, like the inventory: every context loads the WHOLE inventory, then
//   ctx[r].CommInitLocal(r, world); ctx[r].SetShardMap(bounds, strayRank); ctx[r].ShardExport(nOutMax);
//   ctx[r].PeerImportLocal(ctxs)
// Per batch: AllocateBatchGlobal on every context (same claims, without waiting for each other), then GatherRead on the one
// whose table is wanted.  The host does no partitioning and no merging (INTEGRATION.md §4).

func (c *Context) CommInitLocal(rank, world int) error {
	if rc := C.dra_comm_init_local(c.h, C.int(rank), C.int(world)); rc != 0 {
		return lastError(c.h)
	}
	return nil
}

// SetShardMap: rank r serves nodes [bounds[r], bounds[r+1]); len(bounds) == world+1.
func (c *Context) SetShardMap(bounds []uint32, strayRank int) error {
	if rc := C.dra_set_shard_map(c.h, (*C.uint32_t)(unsafe.Pointer(&bounds[0])), C.int(strayRank)); rc != 0 {
		return lastError(c.h)
	}
	return nil
}

func (c *Context) ShardExport(nOutMax uint32) error {
	if rc := C.dra_shard_export(c.h, C.uint32_t(nOutMax), 0, nil); rc != 0 {
		return lastError(c.h)
	}
	return nil
}

func (c *Context) PeerImportLocal(ctxs []*Context) error {
	hs := make([]*C.dra_ctx, len(ctxs))
	for i, o := range ctxs {
		hs[i] = o.h
	}
	if rc := C.dra_peer_import_local(c.h, (**C.dra_ctx)(unsafe.Pointer(&hs[0]))); rc != 0 {
		return lastError(c.h)
	}
	return nil
}

// AllocateBatchGlobal: claims must live in memory from dra_host_alloc (pinned): the device-side range filter then reads them
// over PCIe itself.  Returns at once; GatherRead synchronises.
func (c *Context) AllocateBatchGlobal(pinnedClaims unsafe.Pointer, nClaim int, nOut int, flags uint32) error {
	c.mu.Lock()
	defer c.mu.Unlock()
	rc := C.dra_allocate_batch_global_device(c.h, (*C.dra_claim_rec)(pinnedClaims), C.uint32_t(nClaim), nil, C.uint32_t(nOut), C.uint32_t(flags))
	if rc != 0 {
		return lastError(c.h)
	}
	return nil
}

// SetShardPairs reserves room for the sharded UnsuitableNodes bit exchange: before ShardExport, the same on every context.
// Unbuilt, like the rest of this file.
func (c *Context) SetShardPairs(maxPairs uint32) error {
	if rc := C.dra_set_shard_pairs(c.h, C.uint32_t(maxPairs)); rc != 0 {
		return lastError(c.h)
	}
	return nil
}

// UnsuitableNodesGlobal: UnsuitableNodes on a sharded world (dra_unsuitable_batch_global_device).  The same pods and
// candidates on every context, in dra_host_alloc'ed (pinned) memory; each context decides the pairs of its node range and
// every context ends with the whole bitmap in pinnedBits (ceil(nPair/8) bytes).  candNodes == candOff == nil: dense form,
// nPair = nPod * nNode.  Returns at once; Sync reports completion and errors found on the device.  Unbuilt, like the rest
// of this file.
func (c *Context) UnsuitableNodesGlobal(pinnedClaims unsafe.Pointer, nClaim int, pinnedPodOff unsafe.Pointer, nPod int,
	pinnedCandNodes, pinnedCandOff unsafe.Pointer, nPair int, pinnedBits unsafe.Pointer, flags uint32) error {
	c.mu.Lock()
	defer c.mu.Unlock()
	rc := C.dra_unsuitable_batch_global_device(c.h, (*C.dra_claim_rec)(pinnedClaims), C.uint32_t(nClaim),
		(*C.uint32_t)(pinnedPodOff), C.uint32_t(nPod), (*C.uint32_t)(pinnedCandNodes), (*C.uint32_t)(pinnedCandOff),
		C.uint32_t(nPair), (*C.uint8_t)(pinnedBits), C.uint32_t(flags))
	if rc != 0 {
		return lastError(c.h)
	}
	return nil
}

// AllocatePodsGlobal: pod-mode Allocate on a sharded world (dra_allocate_pods_batch_global_device), the step after
// UnsuitableNodesGlobal with DRA_F_EXHAUSTIVE.  The same pods on every context, in dra_host_alloc'ed (pinned) memory
// (pinnedOutOff may be nil); each context places the pods whose first claim names one of its nodes, and GatherRead gives
// every context the whole table.  Returns at once; Sync reports completion and errors found on the device.  Unbuilt,
// like the rest of this file.
func (c *Context) AllocatePodsGlobal(pinnedClaims unsafe.Pointer, nClaim int, pinnedPodOff unsafe.Pointer, nPod int,
	pinnedOutOff unsafe.Pointer, nOut int, flags uint32) error {
	c.mu.Lock()
	defer c.mu.Unlock()
	rc := C.dra_allocate_pods_batch_global_device(c.h, (*C.dra_claim_rec)(pinnedClaims), C.uint32_t(nClaim),
		(*C.uint32_t)(pinnedPodOff), C.uint32_t(nPod), (*C.uint32_t)(pinnedOutOff), C.uint32_t(nOut), C.uint32_t(flags))
	if rc != 0 {
		return lastError(c.h)
	}
	return nil
}

// SetShardPlace reserves room for the sharded place-pods call's replicated pod states (8 bytes per pod): before
// ShardExport, the same on every context.  Unbuilt, like the rest of this file.
func (c *Context) SetShardPlace(maxPods uint32) error {
	if rc := C.dra_set_shard_place(c.h, C.uint32_t(maxPods)); rc != 0 {
		return lastError(c.h)
	}
	return nil
}

// PlacePodsGlobal: place pods (spec §13) on a sharded world (dra_place_pods_batch_global_device).  The same pods and
// candidates on every context, in dra_host_alloc'ed (pinned) memory (pinnedCandNodes == pinnedCandOff == nil and nPair == 0:
// dense form; pinnedOutOff may be nil); each context evaluates the visits to its own nodes, and every context ends with the
// whole table (GatherRead) and the whole pinnedPodNode (nPod uint32).  Returns at once; Sync reports completion and errors
// found on the device.  Unbuilt, like the rest of this file.
func (c *Context) PlacePodsGlobal(pinnedClaims unsafe.Pointer, nClaim int, pinnedPodOff unsafe.Pointer, nPod int,
	pinnedCandNodes, pinnedCandOff unsafe.Pointer, nPair int, pinnedOutOff unsafe.Pointer, nOut int, pinnedPodNode unsafe.Pointer,
	flags uint32) error {
	c.mu.Lock()
	defer c.mu.Unlock()
	rc := C.dra_place_pods_batch_global_device(c.h, (*C.dra_claim_rec)(pinnedClaims), C.uint32_t(nClaim),
		(*C.uint32_t)(pinnedPodOff), C.uint32_t(nPod), (*C.uint32_t)(pinnedCandNodes), (*C.uint32_t)(pinnedCandOff),
		C.uint32_t(nPair), (*C.uint32_t)(pinnedOutOff), C.uint32_t(nOut), (*C.uint32_t)(pinnedPodNode), C.uint32_t(flags))
	if rc != 0 {
		return lastError(c.h)
	}
	return nil
}

// SetShardPreempt reserves room for the sharded preemption call's per-pod partials and pair results: before ShardExport,
// the same on every context.  Unbuilt, like the rest of this file.
func (c *Context) SetShardPreempt(maxPods, maxPairs, maxVictims uint32) error {
	if rc := C.dra_set_shard_preempt(c.h, C.uint32_t(maxPods), C.uint32_t(maxPairs), C.uint32_t(maxVictims)); rc != 0 {
		return lastError(c.h)
	}
	return nil
}

// PinnedRunningPods: the running pods of PreemptBatchGlobalDevice, every array in dra_host_alloc'ed (pinned) or device
// memory (OutOff may be nil: slot i).
type PinnedRunningPods struct {
	Claims unsafe.Pointer
	NClaim int
	PodOff unsafe.Pointer
	NPod   int
	Prio   unsafe.Pointer
	OutOff unsafe.Pointer
	Out    unsafe.Pointer
	NOut   int
}

// PreemptBatchGlobalDevice: preemption (spec §14) on a sharded world (dra_preempt_batch_global_device).  The same pending
// pods, candidates (pinnedCandNodes == pinnedCandOff == nil: dense form, nPair = nPod * nNode), running pods, maxVictims
// and flags on every context, every array in dra_host_alloc'ed (pinned) memory; each context judges the pairs of its own
// nodes, and every context ends with the whole outputs (the pair outputs may be nil).  Returns at once; Sync reports
// completion and errors found on the device.  Unbuilt, like the rest of this file.
func (c *Context) PreemptBatchGlobalDevice(pinnedClaims unsafe.Pointer, nClaim int, pinnedPodOff, pinnedPrio unsafe.Pointer,
	nPod int, pinnedCandNodes, pinnedCandOff unsafe.Pointer, nPair int, run PinnedRunningPods,
	pinnedPairStatus, pinnedPairVictims, pinnedPodNode, pinnedPodStatus, pinnedNVictims, pinnedVictims unsafe.Pointer,
	maxVictims int, flags uint32) error {
	c.mu.Lock()
	defer c.mu.Unlock()
	var r C.dra_running_pods
	r.claims = (*C.dra_claim_rec)(run.Claims)
	r.n_claim = C.uint32_t(run.NClaim)
	r.pod_off = (*C.uint32_t)(run.PodOff)
	r.n_pod = C.uint32_t(run.NPod)
	r.prio = (*C.int32_t)(run.Prio)
	r.out_off = (*C.uint32_t)(run.OutOff)
	r.out = (*C.dra_out_rec)(run.Out)
	r.n_out = C.uint32_t(run.NOut)
	rc := C.dra_preempt_batch_global_device(c.h, (*C.dra_claim_rec)(pinnedClaims), C.uint32_t(nClaim),
		(*C.uint32_t)(pinnedPodOff), (*C.int32_t)(pinnedPrio), C.uint32_t(nPod), (*C.uint32_t)(pinnedCandNodes),
		(*C.uint32_t)(pinnedCandOff), C.uint32_t(nPair), &r, (*C.uint8_t)(pinnedPairStatus), (*C.uint32_t)(pinnedPairVictims),
		(*C.uint32_t)(pinnedPodNode), (*C.uint8_t)(pinnedPodStatus), (*C.uint32_t)(pinnedNVictims), (*C.uint32_t)(pinnedVictims),
		C.uint32_t(maxVictims), C.uint32_t(flags))
	if rc != 0 {
		return lastError(c.h)
	}
	return nil
}

// PinnedDisruptionBudgets: the budgets of PreemptPdbBatchGlobalDevice in dra_host_alloc'ed (pinned) or device memory.
type PinnedDisruptionBudgets struct {
	RunPdb  unsafe.Pointer
	Allowed unsafe.Pointer
	NPdb    int
}

// PreemptPdbBatchGlobalDevice is PreemptBatchGlobalDevice honouring PodDisruptionBudgets
// (dra_preempt_pdb_batch_global_device), the same budgets on every context; the violation outputs may be nil.  Returns at
// once; Sync reports completion and errors found on the device.  Unbuilt, like the rest of this file.
func (c *Context) PreemptPdbBatchGlobalDevice(pinnedClaims unsafe.Pointer, nClaim int, pinnedPodOff, pinnedPrio unsafe.Pointer,
	nPod int, pinnedCandNodes, pinnedCandOff unsafe.Pointer, nPair int, run PinnedRunningPods, budgets PinnedDisruptionBudgets,
	pinnedPairStatus, pinnedPairVictims, pinnedPairViolations, pinnedPodNode, pinnedPodStatus, pinnedNVictims,
	pinnedPodViolations, pinnedVictims unsafe.Pointer, maxVictims int, flags uint32) error {
	c.mu.Lock()
	defer c.mu.Unlock()
	var r C.dra_running_pods
	r.claims = (*C.dra_claim_rec)(run.Claims)
	r.n_claim = C.uint32_t(run.NClaim)
	r.pod_off = (*C.uint32_t)(run.PodOff)
	r.n_pod = C.uint32_t(run.NPod)
	r.prio = (*C.int32_t)(run.Prio)
	r.out_off = (*C.uint32_t)(run.OutOff)
	r.out = (*C.dra_out_rec)(run.Out)
	r.n_out = C.uint32_t(run.NOut)
	b := C.dra_disruption_budgets{run_pdb: (*C.uint32_t)(budgets.RunPdb), allowed: (*C.int32_t)(budgets.Allowed),
		n_pdb: C.uint32_t(budgets.NPdb)}
	rc := C.dra_preempt_pdb_batch_global_device(c.h, (*C.dra_claim_rec)(pinnedClaims), C.uint32_t(nClaim),
		(*C.uint32_t)(pinnedPodOff), (*C.int32_t)(pinnedPrio), C.uint32_t(nPod), (*C.uint32_t)(pinnedCandNodes),
		(*C.uint32_t)(pinnedCandOff), C.uint32_t(nPair), &r, &b, (*C.uint8_t)(pinnedPairStatus),
		(*C.uint32_t)(pinnedPairVictims), (*C.uint32_t)(pinnedPairViolations), (*C.uint32_t)(pinnedPodNode),
		(*C.uint8_t)(pinnedPodStatus), (*C.uint32_t)(pinnedNVictims), (*C.uint32_t)(pinnedPodViolations),
		(*C.uint32_t)(pinnedVictims), C.uint32_t(maxVictims), C.uint32_t(flags))
	if rc != 0 {
		return lastError(c.h)
	}
	return nil
}

// SetShardCapacity reserves room for the sharded pod-capacity call's pair results: before ShardExport, the same on every
// context.  Unbuilt, like the rest of this file.
func (c *Context) SetShardCapacity(maxPairs uint32) error {
	if rc := C.dra_set_shard_capacity(c.h, C.uint32_t(maxPairs)); rc != 0 {
		return lastError(c.h)
	}
	return nil
}

// PodCapacityBatchGlobalDevice: pod capacity (spec §16) on a sharded world (dra_pod_capacity_batch_global_device).  The
// same pods, candidates (pinnedCandNodes == pinnedCandOff == nil: dense form, nPair = nPod * nNode), maxCopies and flags
// on every context, every array in dra_host_alloc'ed (pinned) memory; each context counts the pairs of its own nodes, and
// every context ends with the whole outputs (all but pinnedPairCopies may be nil).  Returns at once; Sync reports
// completion and errors found on the device.  Unbuilt, like the rest of this file.
func (c *Context) PodCapacityBatchGlobalDevice(pinnedClaims unsafe.Pointer, nClaim int, pinnedPodOff unsafe.Pointer, nPod int,
	pinnedCandNodes, pinnedCandOff unsafe.Pointer, nPair int, maxCopies int,
	pinnedPairCopies, pinnedPairStop, pinnedPodTotal, pinnedPodNodes unsafe.Pointer, flags uint32) error {
	c.mu.Lock()
	defer c.mu.Unlock()
	rc := C.dra_pod_capacity_batch_global_device(c.h, (*C.dra_claim_rec)(pinnedClaims), C.uint32_t(nClaim),
		(*C.uint32_t)(pinnedPodOff), C.uint32_t(nPod), (*C.uint32_t)(pinnedCandNodes), (*C.uint32_t)(pinnedCandOff),
		C.uint32_t(nPair), C.uint32_t(maxCopies), (*C.uint16_t)(pinnedPairCopies), (*C.uint8_t)(pinnedPairStop),
		(*C.uint64_t)(pinnedPodTotal), (*C.uint32_t)(pinnedPodNodes), C.uint32_t(flags))
	if rc != 0 {
		return lastError(c.h)
	}
	return nil
}

// SetShardWhy reserves room for the sharded reasons call's pair records: before ShardExport, the same on every context.
// Unbuilt, like the rest of this file.
func (c *Context) SetShardWhy(maxPairs uint32) error {
	if rc := C.dra_set_shard_why(c.h, C.uint32_t(maxPairs)); rc != 0 {
		return lastError(c.h)
	}
	return nil
}

// PlacePodsWhyBatch places exactly as PlacePodsBatch and also says why each pod went where it did, or nowhere
// (dra_place_pods_why_batch, spec §18): every (pod, candidate) pair answered with a reason and a blocking claim on the
// state the pods before it left, laid out as UnsuitableWhyBatch's (cands == candOff == nil: every node, ascending,
// nNode of them).  Returns the OutRecs, per pod the node it was placed on (0xFFFFFFFF: none), and the reasons.  Unbuilt,
// like the rest of this file.
func (c *Context) PlacePodsWhyBatch(claims []ClaimRec, podOff []uint32, cands, candOff []uint32, nNode int, outOff []uint32,
	nOut int, flags uint32) ([]OutRec, []uint32, *UnsuitableWhy, error) {
	out := make([]OutRec, nOut)
	nPod := len(podOff) - 1
	if nPod <= 0 {
		return out, []uint32{}, &UnsuitableWhy{}, nil
	}
	podNode := make([]uint32, nPod)
	nPair := nPod * nNode
	var cp *C.dra_claim_rec
	var oo, cn, co *C.uint32_t
	if len(claims) > 0 {
		cp = (*C.dra_claim_rec)(unsafe.Pointer(&claims[0]))
	}
	if outOff != nil {
		oo = (*C.uint32_t)(unsafe.Pointer(&outOff[0]))
	}
	if candOff != nil {
		nPair = int(candOff[nPod])
		co = (*C.uint32_t)(unsafe.Pointer(&candOff[0]))
		if len(cands) == 0 {
			cands = []uint32{0} // an empty list still needs an address (nil means the dense form)
		}
		cn = (*C.uint32_t)(unsafe.Pointer(&cands[0]))
	}
	var op *C.dra_out_rec
	if nOut > 0 {
		op = (*C.dra_out_rec)(unsafe.Pointer(&out[0]))
	}
	r := &UnsuitableWhy{make([]uint8, nPair+1), make([]uint32, nPair+1), make([]uint32, nPod*9), make([]uint32, len(claims)+1)}
	c.mu.Lock()
	defer c.mu.Unlock()
	rc := C.dra_place_pods_why_batch(c.h, cp, C.uint32_t(len(claims)), (*C.uint32_t)(unsafe.Pointer(&podOff[0])),
		C.uint32_t(nPod), cn, co, oo, op, C.uint32_t(nOut), (*C.uint32_t)(unsafe.Pointer(&podNode[0])),
		(*C.uint8_t)(unsafe.Pointer(&r.PairWhy[0])), (*C.uint32_t)(unsafe.Pointer(&r.PairClaim[0])),
		(*C.uint32_t)(unsafe.Pointer(&r.PodWhy[0])), (*C.uint32_t)(unsafe.Pointer(&r.ClaimBlocks[0])), C.uint32_t(flags))
	if rc != 0 {
		return nil, nil, nil, lastError(c.h)
	}
	r.PairWhy, r.PairClaim, r.ClaimBlocks = r.PairWhy[:nPair], r.PairClaim[:nPair], r.ClaimBlocks[:len(claims)]
	return out, podNode, r, nil
}

// UnsuitableWhyBatchGlobalDevice: why each node is unsuitable (spec §17) on a sharded world
// (dra_unsuitable_why_batch_global_device).  The same pods, candidates (pinnedCandNodes == pinnedCandOff == nil: dense
// form, nPair = nPod * nNode) and flags on every context, every array in dra_host_alloc'ed (pinned) memory; each context
// judges the pairs of its own nodes, and every context ends with the whole outputs (all but pinnedPairWhy may be nil).
// Returns at once; Sync reports completion and errors found on the device.  Unbuilt, like the rest of this file.
func (c *Context) UnsuitableWhyBatchGlobalDevice(pinnedClaims unsafe.Pointer, nClaim int, pinnedPodOff unsafe.Pointer, nPod int,
	pinnedCandNodes, pinnedCandOff unsafe.Pointer, nPair int,
	pinnedPairWhy, pinnedPairClaim, pinnedPodWhy, pinnedClaimBlocks unsafe.Pointer, flags uint32) error {
	c.mu.Lock()
	defer c.mu.Unlock()
	rc := C.dra_unsuitable_why_batch_global_device(c.h, (*C.dra_claim_rec)(pinnedClaims), C.uint32_t(nClaim),
		(*C.uint32_t)(pinnedPodOff), C.uint32_t(nPod), (*C.uint32_t)(pinnedCandNodes), (*C.uint32_t)(pinnedCandOff),
		C.uint32_t(nPair), (*C.uint8_t)(pinnedPairWhy), (*C.uint32_t)(pinnedPairClaim), (*C.uint32_t)(pinnedPodWhy),
		(*C.uint32_t)(pinnedClaimBlocks), C.uint32_t(flags))
	if rc != 0 {
		return lastError(c.h)
	}
	return nil
}

// PlacePodsWhyBatchGlobalDevice: place pods with reasons (spec §18) on a sharded world
// (dra_place_pods_why_batch_global_device).  The same pods, candidates (pinnedCandNodes == pinnedCandOff == nil and
// nPair == 0: dense form, nPod * nNode pairs answered), outOff, nOut and flags on every context, every array in
// dra_host_alloc'ed (pinned) memory; each context walks the visits to its own nodes, and every context ends with the
// whole table (GatherRead), the whole pod_node and the whole reason outputs (all but pinnedPairWhy may be nil).  Needs
// SetShardPlace and SetShardWhy before ShardExport at world > 1.  Returns at once; Sync reports completion and errors
// found on the device.  Unbuilt, like the rest of this file.
func (c *Context) PlacePodsWhyBatchGlobalDevice(pinnedClaims unsafe.Pointer, nClaim int, pinnedPodOff unsafe.Pointer, nPod int,
	pinnedCandNodes, pinnedCandOff unsafe.Pointer, nPair int, pinnedOutOff unsafe.Pointer, nOut int, pinnedPodNode unsafe.Pointer,
	pinnedPairWhy, pinnedPairClaim, pinnedPodWhy, pinnedClaimBlocks unsafe.Pointer, flags uint32) error {
	c.mu.Lock()
	defer c.mu.Unlock()
	rc := C.dra_place_pods_why_batch_global_device(c.h, (*C.dra_claim_rec)(pinnedClaims), C.uint32_t(nClaim),
		(*C.uint32_t)(pinnedPodOff), C.uint32_t(nPod), (*C.uint32_t)(pinnedCandNodes), (*C.uint32_t)(pinnedCandOff),
		C.uint32_t(nPair), (*C.uint32_t)(pinnedOutOff), C.uint32_t(nOut), (*C.uint32_t)(pinnedPodNode),
		(*C.uint8_t)(pinnedPairWhy), (*C.uint32_t)(pinnedPairClaim), (*C.uint32_t)(pinnedPodWhy),
		(*C.uint32_t)(pinnedClaimBlocks), C.uint32_t(flags))
	if rc != 0 {
		return lastError(c.h)
	}
	return nil
}

// SetShardPreemptPlace reserves room for the sharded preempt-and-place call (pending pods, judged pairs, running pods):
// after SetInventory, before ShardExport, the same on every context.  Unbuilt, like the rest of this file.
func (c *Context) SetShardPreemptPlace(maxPods, maxPairs, maxRun uint32) error {
	if rc := C.dra_set_shard_preempt_place(c.h, C.uint32_t(maxPods), C.uint32_t(maxPairs), C.uint32_t(maxRun)); rc != 0 {
		return lastError(c.h)
	}
	return nil
}

// PreemptPlaceGlobal: preempt and place (spec §15) on a sharded world (dra_preempt_place_batch_global_device).  The same
// pending pods, candidates (pinnedCandNodes == pinnedCandOff == nil and nPair == 0: dense form), running pods, out_off,
// nOut and flags on every context, every array in dra_host_alloc'ed (pinned) memory.  Every context ends with the whole
// table (GatherRead), pod_node, pod_status and evicted_by; the victims are released by the call on the contexts that own
// them.  Returns at once; Sync reports completion and errors found on the device.  Unbuilt, like the rest of this file.
func (c *Context) PreemptPlaceGlobal(pinnedClaims unsafe.Pointer, nClaim int, pinnedPodOff, pinnedPrio unsafe.Pointer,
	nPod int, pinnedCandNodes, pinnedCandOff unsafe.Pointer, nPair int, run PinnedRunningPods, pinnedOutOff unsafe.Pointer,
	nOut int, pinnedPodNode, pinnedPodStatus, pinnedEvictedBy unsafe.Pointer, flags uint32) error {
	c.mu.Lock()
	defer c.mu.Unlock()
	var r C.dra_running_pods
	r.claims = (*C.dra_claim_rec)(run.Claims)
	r.n_claim = C.uint32_t(run.NClaim)
	r.pod_off = (*C.uint32_t)(run.PodOff)
	r.n_pod = C.uint32_t(run.NPod)
	r.prio = (*C.int32_t)(run.Prio)
	r.out_off = (*C.uint32_t)(run.OutOff)
	r.out = (*C.dra_out_rec)(run.Out)
	r.n_out = C.uint32_t(run.NOut)
	rc := C.dra_preempt_place_batch_global_device(c.h, (*C.dra_claim_rec)(pinnedClaims), C.uint32_t(nClaim),
		(*C.uint32_t)(pinnedPodOff), (*C.int32_t)(pinnedPrio), C.uint32_t(nPod), (*C.uint32_t)(pinnedCandNodes),
		(*C.uint32_t)(pinnedCandOff), C.uint32_t(nPair), &r, (*C.uint32_t)(pinnedOutOff), C.uint32_t(nOut),
		(*C.uint32_t)(pinnedPodNode), (*C.uint8_t)(pinnedPodStatus), (*C.uint32_t)(pinnedEvictedBy), C.uint32_t(flags))
	if rc != 0 {
		return lastError(c.h)
	}
	return nil
}

// DeallocateGlobal: Deallocate on a sharded world (dra_deallocate_batch_global_device), the step after AllocatePodsGlobal.
// The same claims, out_off and OutRecs on every context, in dra_host_alloc'ed (pinned) memory (pinnedOutOff may be nil);
// each context applies the OK records whose GPU lies in its own range and writes no other GPU.  Needs SetShardMap (or
// SetShard) after SetInventory, and no export, import or peer.  A slot range outside nOut fails the call at Sync on every
// context with no inventory changed.  Returns at once; Sync reports completion and errors found on the device.  Unbuilt,
// like the rest of this file.
func (c *Context) DeallocateGlobal(pinnedClaims unsafe.Pointer, nClaim int, pinnedOutOff unsafe.Pointer, pinnedOut unsafe.Pointer,
	nOut int) error {
	c.mu.Lock()
	defer c.mu.Unlock()
	rc := C.dra_deallocate_batch_global_device(c.h, (*C.dra_claim_rec)(pinnedClaims), C.uint32_t(nClaim),
		(*C.uint32_t)(pinnedOutOff), (*C.dra_out_rec)(pinnedOut), C.uint32_t(nOut))
	if rc != 0 {
		return lastError(c.h)
	}
	return nil
}

// ShardSyncInventory makes every context's live inventory the world's state (dra_shard_sync_inventory_device): each GPU's
// record as the context owning its node holds it.  Afterwards dra_get_inventory on any context returns the whole world,
// and SetShardMap may move node ranges without losing allocations.  Every context must make the call; needs SetShardMap
// and ShardExport after SetInventory, then PeerImportLocal.  One process: call it on EVERY context before SetShardMap or
// dra_get_inventory on any, since both wait for the context's stream.  Returns at once; Sync reports completion and errors found
// on the device.  Unbuilt, like the rest of this file.
func (c *Context) ShardSyncInventory() error {
	c.mu.Lock()
	defer c.mu.Unlock()
	if rc := C.dra_shard_sync_inventory_device(c.h); rc != 0 {
		return lastError(c.h)
	}
	return nil
}

// Sync waits for the calls enqueued on the context and reports the errors they found on the device (dra_ctx_sync).
func (c *Context) Sync() error {
	c.mu.Lock()
	defer c.mu.Unlock()
	if rc := C.dra_ctx_sync(c.h); rc != 0 {
		return lastError(c.h)
	}
	return nil
}

func (c *Context) GatherRead(out []OutRec) error {
	c.mu.Lock()
	defer c.mu.Unlock()
	if rc := C.dra_gather_read(c.h, (*C.dra_out_rec)(unsafe.Pointer(&out[0])), C.uint32_t(len(out))); rc != 0 {
		return lastError(c.h)
	}
	return nil
}

// PeerRendezvous lines the contexts' streams up on the device (optional; dra_peer_rendezvous_device).
func (c *Context) PeerRendezvous() error {
	if rc := C.dra_peer_rendezvous_device(c.h); rc != 0 {
		return lastError(c.h)
	}
	return nil
}
