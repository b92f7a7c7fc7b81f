// Package mpi is the drop-in facade for github.com/btracey/mpi on a box of NVIDIA H100 GPUs.
//
// UNVERIFIED: this image has no Go toolchain, so these files have never been compiled.  They are
// the binding a maintainer adds; the C ABI they call (include/b200mpi.h) is exercised end to end
// by the C++ facade (mpi_b200/cpp/mpi.hpp) and by the Python harness through the same entry points.
//
// Callers keep writing
//
//	flag.Parse(); mpi.Init(); defer mpi.Finalize()
//	mpi.Send(x, dst, tag); mpi.Receive(&y, src, tag)
//
// exactly as with the reference (function set and signatures of reference mpi.go:96-159, the
// Interface of mpi.go:163-170, Register of mpi.go:61-67, Raw of mpi.go:75-91, TagExists of
// mpi.go:174-182).  What changes is the default implementation behind the facade: instead of
// Network (gob over TCP, network.go) it is Cuda (cuda.go), a cgo layer over libb200mpi.so whose
// kernels move the slices between GPUs through NVSwitch peer memory.
//
// New entry points, following the same conventions (package function forwarding to the
// registered implementation, blocking, error return, data typed by its Go slice type):
//
//	Recv       alias of Receive (the reference spells it Receive)
//	Bcast      root's slice to every rank
//	Allreduce  element-wise reduction over ranks, result on every rank
//	Allgather  concatenation in rank order on every rank
//	Barrier    rendezvous of all ranks
//	ReduceScatter, Reduce, Alltoall   the usual MPI companions of the above
//	Gather, Scatter                   rooted collection and distribution of equal blocks
//	Gatherv, Scatterv, Allgatherv     the same with a different length on every rank
//	Alltoallv                         Alltoall with a different length for every (source, destination) pair
//	Scan, Exscan                      prefix reductions in rank order (inclusive, exclusive)
//	ReduceScatterv                    ReduceScatter with a different block length for every rank
//	AllreduceLoc, ReduceLoc           MAXLOC / MINLOC: the best value across ranks and where it came from
//	WinCreate -> Window               one-sided Put, Get and Accumulate into other ranks' heap memory, completed by Fence
//	PassiveWindow                     Lock, Unlock, GetAccumulate, FetchAndOp, CompareAndSwap (type-assert the Window)
//	GroupWindow                       Post, Start, Complete, Wait, Test: epochs between named ranks only (type-assert the Window)
//	Isend + Wait   the non-blocking Send design the reference sketches and comments out (mpi.go:132-152)
//
// They are served through the optional Collective interface, the upgrade the reference hints at
// with its unused isAllReducer variable (mpi.go:69-71).
package mpi

import "fmt"

// Interface is the set of routines an implementation must provide; unchanged from the reference.
type Interface interface {
	Init() error
	Finalize()
	Rank() int
	Size() int
	Send(data interface{}, destination, tag int) error
	Receive(data interface{}, source, tag int) error
}

// Op selects the reduction of Allreduce.
type Op int

const (
	Sum Op = iota
	Max
	Min
	Replace // one-sided calls only: the target takes origin's value
	NoOp    // GetAccumulate and FetchAndOp only: the target is left as it is (an atomic read)
)

// LockType selects the lock PassiveWindow.Lock takes on a target's window.
type LockType int

const (
	LockExclusive LockType = 1 // excludes every other holder
	LockShared    LockType = 2 // excludes exclusive holders only
)

// Collective is implemented by transports that offer collectives natively.
type Collective interface {
	Bcast(data interface{}, root int) error
	Allreduce(send, recv interface{}, op Op) error
	Allgather(send, recv interface{}) error
	Barrier() error
}

// Collective2 is the second optional upgrade: further collectives and the Isend/Wait pair.
type Collective2 interface {
	ReduceScatter(send, recv interface{}, op Op) error
	Reduce(send, recv interface{}, op Op, root int) error
	Alltoall(send, recv interface{}) error
	Isend(data interface{}, destination, tag int) error
	Wait(destination, tag int) error
}

// Collective3 is the third optional upgrade: the rooted and variable-count collectives. Receivers
// are pointers to slices, resized the way Receive resizes (or a *DeviceSlice of the right length).
// counts is the same table on every rank; a nil counts is learnt (see Gatherv, Scatterv) and the
// table used is returned.
type Collective3 interface {
	Gather(send, recv interface{}, root int) error
	Scatter(send, recv interface{}, root int) error
	Gatherv(send, recv interface{}, counts []int, root int) ([]int, error)
	Scatterv(send, recv interface{}, counts []int, root int) ([]int, error)
	Allgatherv(send, recv interface{}, counts []int) ([]int, error)
}

// Collective4 is the fourth optional upgrade: the variable-count exchange. Unlike Collective3's
// tables, sendCounts and recvCounts are this rank's own row and column and differ from rank to rank.
type Collective4 interface {
	Alltoallv(send interface{}, sendCounts []int, recv interface{}, recvCounts []int) ([]int, error)
}

// Collective5 is the fifth optional upgrade: the prefix reductions.
type Collective5 interface {
	Scan(send, recv interface{}, op Op) error
	Exscan(send, recv interface{}, op Op) error
}

// Collective6 is the sixth optional upgrade: the reduce-scatter whose blocks follow a counts table.
type Collective6 interface {
	ReduceScatterv(send, recv interface{}, counts []int, op Op) ([]int, error)
}

// Collective7 is the seventh optional upgrade: the value-location reductions (MPI's MAXLOC and
// MINLOC). op is Max or Min.
type Collective7 interface {
	AllreduceLoc(send, recv interface{}, op Op) error
	ReduceLoc(send, recv interface{}, op Op, root int) error
}

// Collective8 is the eighth optional upgrade: one-sided communication (MPI-3 active target with
// fence synchronisation) through windows of every rank's device heap.
type Collective8 interface {
	WinCreate(local *DeviceSlice) (Window, error)
}

// Window is memory of every rank's heap that any rank may Put into, Get from and Accumulate into.
// origin is a []float64, []float32, []int64, []byte or *DeviceSlice; disp counts elements of the
// origin's type from the start of rank target's window, and the range must fit in it. Each call
// returns once origin may be reused (Get: once it holds the data). What Put and Accumulate write is
// visible to the target after its next Fence, which every rank calls; a location written by one
// rank and read or written by another between two fences is undefined, except by Accumulates with
// the same type and op. Accumulate (Sum, Max, Min over float32, float64 and int64) is element-wise
// atomic: int64 Sum wraps, float32 Sum flushes subnormal values to zero, float Max and Min keep a NaN
// already in the target and ignore a NaN in origin. Free is a Fence that also drops the window.
type Window interface {
	Put(origin interface{}, target, disp int) error
	Get(origin interface{}, target, disp int) error
	Accumulate(origin interface{}, target, disp int, op Op) error
	Fence() error
	Free() error
}

// PassiveWindow is a Window with passive-target synchronisation and atomic fetches (MPI-3). Window
// itself is unchanged, so other implementations of it still compile; reach these with a type
// assertion, w.(PassiveWindow). None of them is collective.
//
// Lock blocks until this rank holds the lock on rank target's window (target may be this rank); it
// fails with a timeout after the watchdog_ms knob, holding nothing. There is no fairness. Every call
// has completed when it returns, so what this rank did under a lock is visible to the next holder.
// A rank holding a lock on a window must not Fence or Free it: that call fails on every rank.
// GetAccumulate sets result to the target's previous values and applies op (Sum, Max, Min, Replace or
// NoOp, whose origin may be nil), one atomic per element; result has origin's type, length and
// storage, and may be origin itself. FetchAndOp does the same for one float32, float64 or int64 value
// and returns the previous value with its type. CompareAndSwap (int64) returns the previous value and
// stores value if that equalled compare.
type PassiveWindow interface {
	Window
	Lock(target int, lockType LockType) error
	Unlock(target int) error
	GetAccumulate(origin, result interface{}, target, disp int, op Op) error
	FetchAndOp(value interface{}, target, disp int, op Op) (interface{}, error)
	CompareAndSwap(value, compare int64, target, disp int) (int64, error)
}

// GroupWindow is a Window with generalized active-target synchronisation (MPI-3 post / start /
// complete / wait). Window itself is unchanged; reach these with a type assertion, w.(GroupWindow).
// None of them is collective: only the ranks named in the groups take part. A group is a list of
// distinct ranks; it may be empty or include this rank.
//
// Post opens an exposure epoch of this rank's window to origins and does not block. Start opens an
// access epoch to targets and blocks until each has posted to this rank; after the watchdog_ms knob
// it fails with a timeout, and no epoch is open. Complete closes the access epoch. Wait closes the
// exposure epoch once every origin has completed; after watchdog_ms it fails with a timeout and the
// epoch stays open. Test is Wait without waiting: true and closed, or false and still open. What an
// origin put between Start and Complete is visible to the target once Wait returns. A rank with an
// epoch open on a window must not Fence or Free it: that call fails on every rank.
type GroupWindow interface {
	Window
	Post(origins []int) error
	Start(targets []int) error
	Complete() error
	Wait() error
	Test() (bool, error)
}

// Float32Loc, Float64Loc and Int64Loc are the elements of AllreduceLoc and ReduceLoc: a value and
// where it came from. Each is 16 bytes, the layout of the C struct { V val; int64_t loc; } (4
// padding bytes follow a float32).
type Float32Loc struct {
	Val float32
	Loc int64
}

type Float64Loc struct {
	Val float64
	Loc int64
}

type Int64Loc struct {
	Val int64
	Loc int64
}

// Raw marks a payload that is sent as bytes without any encoding.
type Raw []byte

// GobEncode keeps Raw usable with gob-based implementations such as the reference's Network.
func (r Raw) GobEncode() ([]byte, error) { return append([]byte(nil), r...), nil }

// GobDecode is the inverse of GobEncode; it reuses the destination when it is large enough.
func (r *Raw) GobDecode(b []byte) error {
	if cap(*r) >= len(b) {
		*r = (*r)[:len(b)]
	} else {
		*r = make(Raw, len(b))
	}
	copy(*r, b)
	return nil
}

// TagExists reports that {peer, tag} already has a request in flight.
type TagExists struct {
	Tag int
}

func (t TagExists) Error() string { return fmt.Sprintf("Tag %v already in use sending", t.Tag) }

var (
	current    Interface = &Cuda{}
	registered bool
)

// Register installs an implementation; it may be called once, during program initialisation.
func Register(impl Interface) {
	if registered {
		panic("register called more than once")
	}
	current, registered = impl, true
}

// Init must precede every other call. flag.Parse() must have run if the -mpi-* flags are used.
func Init() error { return current.Init() }

// Finalize ends the session; no call may follow it.
func Finalize() { current.Finalize() }

// Rank is this process's index in the sorted address list, or -1 before Init.
func Rank() int { return current.Rank() }

// Size is the number of ranks, or 0 before Init.
func Size() int { return current.Size() }

// Send blocks until the matching Receive has taken the data. Concurrent calls need distinct
// {destination, tag} pairs.
func Send(data interface{}, destination, tag int) error {
	return current.Send(data, destination, tag)
}

// Receive blocks for the message {source, tag} and stores it through the pointer data, resizing
// the destination slice to the sent length.
func Receive(data interface{}, source, tag int) error {
	return current.Receive(data, source, tag)
}

// Recv is Receive.
func Recv(data interface{}, source, tag int) error { return Receive(data, source, tag) }

func collective() (Collective, error) {
	if c, ok := current.(Collective); ok {
		return c, nil
	}
	return nil, fmt.Errorf("mpi: registered implementation %T has no collectives", current)
}

// Bcast copies root's slice into data on every rank. data is a slice (or *DeviceSlice).
func Bcast(data interface{}, root int) error {
	c, err := collective()
	if err != nil {
		return err
	}
	return c.Bcast(data, root)
}

// Allreduce reduces send element-wise over all ranks into recv on every rank; send and recv are
// slices of the same type and length ([]float32, []float64, []int64) and may be the same slice.
func Allreduce(send, recv interface{}, op Op) error {
	c, err := collective()
	if err != nil {
		return err
	}
	return c.Allreduce(send, recv, op)
}

// Allgather stores rank r's send at recv[r*len(send):(r+1)*len(send)] on every rank.
func Allgather(send, recv interface{}) error {
	c, err := collective()
	if err != nil {
		return err
	}
	return c.Allgather(send, recv)
}

// Barrier returns once every rank has called it.
func Barrier() error {
	c, err := collective()
	if err != nil {
		return err
	}
	return c.Barrier()
}

func collective2() (Collective2, error) {
	if c, ok := current.(Collective2); ok {
		return c, nil
	}
	return nil, fmt.Errorf("mpi: registered implementation %T has no ReduceScatter/Reduce/Alltoall/Isend", current)
}

// ReduceScatter reduces block j of every rank's send (Size() blocks of len(recv)) into rank j's recv.
func ReduceScatter(send, recv interface{}, op Op) error {
	c, err := collective2()
	if err != nil {
		return err
	}
	return c.ReduceScatter(send, recv, op)
}

// Reduce is Allreduce with the result on root only; recv may be nil on the other ranks.
func Reduce(send, recv interface{}, op Op, root int) error {
	c, err := collective2()
	if err != nil {
		return err
	}
	return c.Reduce(send, recv, op, root)
}

// Alltoall sends block j of send to rank j, where it becomes block Rank() of recv.
func Alltoall(send, recv interface{}) error {
	c, err := collective2()
	if err != nil {
		return err
	}
	return c.Alltoall(send, recv)
}

// Isend transmits data to destination and returns once data may be modified again, without
// waiting for the receiver (the Send of the reference's commented-out design, mpi.go:132-143).
// The {destination, tag} pair stays in use until Wait.
func Isend(data interface{}, destination, tag int) error {
	c, err := collective2()
	if err != nil {
		return err
	}
	return c.Isend(data, destination, tag)
}

// Wait blocks until destination confirmed the message sent with tag, and frees the pair for
// re-use (mpi.go:146-152).
func Wait(destination, tag int) error {
	c, err := collective2()
	if err != nil {
		return err
	}
	return c.Wait(destination, tag)
}

func collective3() (Collective3, error) {
	if c, ok := current.(Collective3); ok {
		return c, nil
	}
	return nil, fmt.Errorf("mpi: registered implementation %T has no Gather/Scatter/Gatherv/Scatterv/Allgatherv", current)
}

// Gather stores rank r's send in block r of root's recv, which is resized to Size()*len(send).
// recv may be nil on the other ranks.
func Gather(send, recv interface{}, root int) error {
	c, err := collective3()
	if err != nil {
		return err
	}
	return c.Gather(send, recv, root)
}

// Scatter sends block r of root's send (Size() equal blocks) to rank r's recv. root's recv is
// resized to one block; the other ranks' recv must already hold that length. send may be nil off root.
func Scatter(send, recv interface{}, root int) error {
	c, err := collective3()
	if err != nil {
		return err
	}
	return c.Scatter(send, recv, root)
}

// Gatherv stores rank r's send at offset counts[0]+...+counts[r-1] of root's recv, resized to
// sum(counts). A nil counts on every rank is learnt with one Allgather of the lengths.
func Gatherv(send, recv interface{}, counts []int, root int) ([]int, error) {
	c, err := collective3()
	if err != nil {
		return nil, err
	}
	return c.Gatherv(send, recv, counts, root)
}

// Scatterv sends root's send[displ[r]:displ[r]+counts[r]] to rank r's recv, resized to counts[r].
// root passes counts; the other ranks may pass nil and learn root's table.
func Scatterv(send, recv interface{}, counts []int, root int) ([]int, error) {
	c, err := collective3()
	if err != nil {
		return nil, err
	}
	return c.Scatterv(send, recv, counts, root)
}

// Allgatherv is Gatherv with the result on every rank.
func Allgatherv(send, recv interface{}, counts []int) ([]int, error) {
	c, err := collective3()
	if err != nil {
		return nil, err
	}
	return c.Allgatherv(send, recv, counts)
}

// Alltoallv sends block j of send (sendCounts[j] elements, packed in rank order) to rank j; the
// block from rank r lands at offset recvCounts[0]+...+recvCounts[r-1] of recv, which is resized to
// sum(recvCounts). recvCounts[r] must equal rank r's sendCounts[Rank()]; a nil recvCounts is learnt
// with one Alltoall of sendCounts, and the table used is returned.
func Alltoallv(send interface{}, sendCounts []int, recv interface{}, recvCounts []int) ([]int, error) {
	c, ok := current.(Collective4)
	if !ok {
		return nil, fmt.Errorf("mpi: registered implementation %T has no Alltoallv", current)
	}
	return c.Alltoallv(send, sendCounts, recv, recvCounts)
}

func collective5(what string) (Collective5, error) {
	if c, ok := current.(Collective5); ok {
		return c, nil
	}
	return nil, fmt.Errorf("mpi: registered implementation %T has no %s", current, what)
}

// Scan stores send_0 op send_1 op ... op send_r, combined in rank order, in rank r's recv. send and
// recv are slices of the same type and length ([]float32, []float64, []int64) and may be the same slice.
func Scan(send, recv interface{}, op Op) error {
	c, err := collective5("Scan")
	if err != nil {
		return err
	}
	return c.Scan(send, recv, op)
}

// Exscan is Scan without rank r's own send: rank r >= 1 receives send_0 op ... op send_{r-1}.
// Rank 0's recv is not written and may be nil. An Exscan of each rank's element count gives its
// offset in a buffer packed in rank order.
func Exscan(send, recv interface{}, op Op) error {
	c, err := collective5("Exscan")
	if err != nil {
		return err
	}
	return c.Exscan(send, recv, op)
}

// ReduceScatterv reduces block j of every rank's send (counts[j] elements at offset
// counts[0]+...+counts[j-1]; send holds sum(counts)) with op, in rank order, into rank j's recv,
// which is resized to counts[j]. A nil counts on every rank is learnt from len(recv) with one
// Allgather, and the table used is returned. In place: recv points at this rank's block of send,
// the form an in-place Allgatherv with the same table completes into an Allreduce.
func ReduceScatterv(send, recv interface{}, counts []int, op Op) ([]int, error) {
	c, ok := current.(Collective6)
	if !ok {
		return nil, fmt.Errorf("mpi: registered implementation %T has no ReduceScatterv", current)
	}
	return c.ReduceScatterv(send, recv, counts, op)
}

func collective7(what string) (Collective7, error) {
	if c, ok := current.(Collective7); ok {
		return c, nil
	}
	return nil, fmt.Errorf("mpi: registered implementation %T has no %s", current, what)
}

// AllreduceLoc combines, pair by pair and in rank order, every rank's send ([]Float32Loc,
// []Float64Loc or []Int64Loc) into every rank's recv, a slice of the same type and length (it may be
// send). With op Max (MAXLOC) or Min (MINLOC) a higher rank's pair replaces the running one when its
// value is better, or equal with a smaller Loc. Floats compare as IEEE (-0 == +0), except that NaN is
// better than every number under both ops and equal to every NaN, so NaN propagates as it does with
// math.Max and math.Min. The winning pair is copied whole, so every rank gets the same bytes. Loc is
// usually Rank() or a global index: a MINLOC with Loc = Rank() names the rank to Bcast from.
func AllreduceLoc(send, recv interface{}, op Op) error {
	c, err := collective7("AllreduceLoc")
	if err != nil {
		return err
	}
	return c.AllreduceLoc(send, recv, op)
}

// ReduceLoc is AllreduceLoc whose result lands in root's recv only; recv may be nil elsewhere.
func ReduceLoc(send, recv interface{}, op Op, root int) error {
	c, err := collective7("ReduceLoc")
	if err != nil {
		return err
	}
	return c.ReduceLoc(send, recv, op, root)
}

// WinCreate is collective: every rank exposes local, a *DeviceSlice from Alloc (nil for an empty
// window), to one-sided calls by every rank. Windows may differ in size from rank to rank.
func WinCreate(local *DeviceSlice) (Window, error) {
	c, ok := current.(Collective8)
	if !ok {
		return nil, fmt.Errorf("mpi: registered implementation %T has no WinCreate", current)
	}
	return c.WinCreate(local)
}
